// pb_own.cuh — the C ABI's error reporting and the CUDA resources its objects hold (included by pb_api.cu only).
// Every buffer, mapped pinned host block, shared host mapping, stream-ordered buffer, stream, event and IPC mapping an
// object acquires is
// recorded in its Owned, which releases what is still held, in reverse order, when the object is deleted.  A step that
// acquires several resources acquires them into a local Owned and adopts it once every part has succeeded, then sets
// its gate: a step that fails leaves nothing allocated and no gate set, and the next call acquires afresh.
// A growable table's storage (pb_table_set_growth) is device address space reserved for its whole capacity and backed
// by physical memory chunk by chunk: the reservation and each chunk are resources of their own.
#pragma once
#include <atomic>
#include <cerrno>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cuda.h>  // the driver's types only: its virtual-memory calls are reached through cudaGetDriverEntryPoint
#include <cuda_runtime.h>

#include "persia_b200.h"

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define PB_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return fail(PB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));               \
  } while (0)

// what every live object holds (pb_debug_owned), and the acquisitions still granted before one is refused
// (pb_debug_refuse_after; -1: none is)
std::atomic<uint64_t> g_owned_count{0}, g_owned_bytes{0};
std::atomic<int64_t> g_refuse_after{-1};

// The driver's virtual-memory calls, looked up once through the runtime, so that the library links only the shared
// cudart.  `ok` false: the driver lacks one of them (every growable table is then refused).
struct Vmm {
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemAddressFree) free = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemSetAccess) access = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  bool ok = false;
};

const Vmm& vmm() {
  static const Vmm v = [] {
    Vmm w;
    auto get = [](const char* name, auto& fn) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
      if (cudaGetDriverEntryPointByVersion(name, &p, 12000, cudaEnableDefault, &q) != cudaSuccess ||
          q != cudaDriverEntryPointSuccess)
        p = nullptr;
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(p);
      return p != nullptr;
    };
    w.ok = get("cuMemAddressReserve", w.reserve) & get("cuMemAddressFree", w.free) & get("cuMemCreate", w.create) &
           get("cuMemRelease", w.release) & get("cuMemMap", w.map) & get("cuMemUnmap", w.unmap) &
           get("cuMemSetAccess", w.access) & get("cuMemGetAllocationGranularity", w.granularity);
    return w;
  }();
  return v;
}

CUmemAllocationProp vmm_prop(int device) {
  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  return prop;
}

// the size every chunk of `device` is a multiple of (0: no virtual-memory support)
size_t vmm_granularity(int device) {
  const Vmm& v = vmm();
  size_t g = 0;
  const CUmemAllocationProp prop = vmm_prop(device);
  if (!v.ok || v.granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS) return 0;
  return g;
}

struct Owned {
  enum Kind { DEV, HOST, ASYNC, STREAM, EVENT, IPC, SHARED, VRESERVE, VCHUNK };
  struct Res {
    void* p;
    Kind kind;
    size_t bytes;     // counted in pb_debug_owned (a reservation: 0)
    cudaStream_t st;  // ASYNC: the stream it was allocated on (the destructor frees it there)
    int fd = -1;      // SHARED: the file the mapping is of
    size_t span = 0;  // VRESERVE: the address range reserved
    unsigned long long handle = 0;  // VCHUNK: the physical allocation mapped at p
  };
  std::vector<Res> held;

  Owned() = default;
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() {
    while (!held.empty()) drop(held.size() - 1, held.back().st);
  }

  template <typename T>
  int dev(T*& p, size_t bytes) {
    void* q = nullptr;
    const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaMalloc(&q, bytes);
    return keep(e, "cudaMalloc", q, DEV, bytes, nullptr, p);
  }
  // pinned host memory mapped into the device's address space: `h` its host address, `d` its device address
  template <typename T>
  int mapped(T*& h, T*& d, size_t bytes) {
    void *q = nullptr, *dq = nullptr;
    cudaError_t e =
        refused() ? cudaErrorMemoryAllocation : cudaHostAlloc(&q, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (int rc = keep(e, "cudaHostAlloc", q, HOST, bytes, nullptr, q)) return rc;
    if ((e = cudaHostGetDevicePointer(&dq, q, 0)) != cudaSuccess) {
      release(q);
      return fail(PB_ERR_CUDA, std::string("cudaHostGetDevicePointer: ") + cudaGetErrorString(e));
    }
    h = static_cast<T*>(q);
    d = static_cast<T*>(dq);
    return PB_OK;
  }
  // Host memory another process can map (pb_table_create_host_shared): `fd` < 0, a new anonymous memfd of `bytes`;
  // else `fd` itself (a peer's, opened through /proc), whose size must be `bytes`.  The file is mapped MAP_SHARED
  // (populated, not write-combined) and registered mapped into the device's address space: `h` its host address, `d`
  // its device address, `fd_out` the descriptor.  read_only (a peer's, where the device can register read-only memory):
  // mapped PROT_READ and registered cudaHostRegisterReadOnly, so that no stray write of a reader reaches the owner's
  // rows (`fd` then needs no write access).  Released as unregister, unmap, close; a failed step undoes the ones before
  // it, and a given `fd` is closed on failure too.
  template <typename T>
  int shared(T*& h, T*& d, size_t bytes, int fd, int& fd_out, bool read_only = false) {
    if (refused()) {
      if (fd >= 0) close(fd);
      return fail(PB_ERR_CUDA, "shared host mapping: refused");
    }
    const bool created = fd < 0;
    if (created && (fd = memfd_create("persia_b200_tier", MFD_CLOEXEC)) < 0)
      return fail(PB_ERR_CUDA, std::string("memfd_create: ") + strerror(errno));
    struct stat sb;
    const char* what = nullptr;
    errno = 0;
    if (created && ftruncate(fd, (off_t)bytes) != 0) what = "ftruncate";
    else if (!created && (fstat(fd, &sb) != 0 || (size_t)sb.st_size != bytes)) what = "the shared tier's size";
    void* q = MAP_FAILED;
    const int prot = read_only ? PROT_READ : PROT_READ | PROT_WRITE;
    if (!what && (q = mmap(nullptr, bytes, prot, MAP_SHARED | MAP_POPULATE, fd, 0)) == MAP_FAILED) what = "mmap";
    if (what) {
      const std::string msg = std::string(what) + ": " + (errno ? strerror(errno) : "mismatch");
      close(fd);
      return fail(PB_ERR_STATE, msg);
    }
    cudaError_t e = cudaHostRegister(q, bytes, cudaHostRegisterMapped | cudaHostRegisterPortable |
                                                   (read_only ? cudaHostRegisterReadOnly : 0u));
    void* dq = nullptr;
    if (e == cudaSuccess && (e = cudaHostGetDevicePointer(&dq, q, 0)) != cudaSuccess) cudaHostUnregister(q);
    if (e != cudaSuccess) {
      munmap(q, bytes);
      close(fd);
      return fail(PB_ERR_CUDA, std::string("cudaHostRegister: ") + cudaGetErrorString(e));
    }
    held.push_back({q, SHARED, bytes, nullptr, fd});
    g_owned_count += 1;
    g_owned_bytes += bytes;
    h = static_cast<T*>(q);
    d = static_cast<T*>(dq);
    fd_out = fd;
    return PB_OK;
  }
  // stream-ordered: allocated in `st`'s order
  template <typename T>
  int async(T*& p, size_t bytes, cudaStream_t st) {
    void* q = nullptr;
    const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaMallocAsync(&q, bytes, st);
    return keep(e, "cudaMallocAsync", q, ASYNC, bytes, st, p);
  }
  int stream(cudaStream_t& s) {
    cudaStream_t q = nullptr;
    const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking);
    return keep(e, "cudaStreamCreateWithFlags", q, STREAM, 0, nullptr, s);
  }
  int event(cudaEvent_t& ev) {
    cudaEvent_t q = nullptr;
    const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaEventCreateWithFlags(&q, cudaEventDisableTiming);
    return keep(e, "cudaEventCreateWithFlags", q, EVENT, 0, nullptr, ev);
  }
  // `bytes` of device address space, nothing behind it yet (chunk() backs it)
  template <typename T>
  int reserve(T*& p, size_t bytes) {
    const Vmm& v = vmm();
    CUdeviceptr q = 0;
    if (!v.ok) return fail(PB_ERR_CUDA, "the driver lacks the virtual memory management calls");
    if (refused()) return fail(PB_ERR_CUDA, "cuMemAddressReserve: refused");
    if (CUresult e = v.reserve(&q, bytes, 0, 0, 0))
      return fail(PB_ERR_CUDA, "cuMemAddressReserve: CUresult " + std::to_string((int)e));
    held.push_back({reinterpret_cast<void*>(q), VRESERVE, 0, nullptr, -1, bytes, 0});
    g_owned_count += 1;
    p = reinterpret_cast<T*>(q);
    return PB_OK;
  }
  // `bytes` (a multiple of vmm_granularity) of `device`'s memory, created and mapped read-write at `at`, inside a
  // reservation; undone as unmap, release
  int chunk(void* at, size_t bytes, int device) {
    const Vmm& v = vmm();
    const CUmemAllocationProp prop = vmm_prop(device);
    CUmemGenericAllocationHandle h = 0;
    if (refused()) return fail(PB_ERR_CUDA, "cuMemCreate: refused");
    if (CUresult e = v.create(&h, bytes, &prop, 0))
      return fail(PB_ERR_CUDA, "cuMemCreate: CUresult " + std::to_string((int)e));
    const CUdeviceptr q = reinterpret_cast<CUdeviceptr>(at);
    CUresult e = v.map(q, bytes, 0, h, 0);
    if (e == CUDA_SUCCESS) {
      CUmemAccessDesc acc;
      std::memset(&acc, 0, sizeof(acc));
      acc.location = prop.location;
      acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      if ((e = v.access(q, bytes, &acc, 1)) != CUDA_SUCCESS) v.unmap(q, bytes);
    }
    if (e != CUDA_SUCCESS) {
      v.release(h);
      return fail(PB_ERR_CUDA, "cuMemMap / cuMemSetAccess: CUresult " + std::to_string((int)e));
    }
    held.push_back({at, VCHUNK, bytes, nullptr, -1, 0, (unsigned long long)h});
    g_owned_count += 1;
    g_owned_bytes += bytes;
    return PB_OK;
  }
  // another process's allocation, mapped into this one
  int ipc(void*& p, const cudaIpcMemHandle_t& h) {
    void* q = nullptr;
    const cudaError_t e =
        refused() ? cudaErrorMapBufferObjectFailed : cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
    return keep(e, "cudaIpcOpenMemHandle", q, IPC, 0, nullptr, p);
  }

  // Release one resource now and null the caller's pointer (null, or not held here: nothing is released).  A
  // stream-ordered buffer is freed in `st`'s order.
  template <typename T>
  void release(T*& p, cudaStream_t st = nullptr) {
    for (size_t i = held.size(); p && i--;)
      if (held[i].p == static_cast<const void*>(p)) {
        drop(i, st);
        break;
      }
    p = nullptr;
  }
  // release everything, stream-ordered buffers in `st`'s order
  void release_all(cudaStream_t st) {
    while (!held.empty()) drop(held.size() - 1, st);
  }
  // take over what `o` holds (a step that has succeeded)
  void adopt(Owned& o) {
    held.insert(held.end(), o.held.begin(), o.held.end());
    o.held.clear();
  }

 private:
  // pb_debug_refuse_after: this acquisition is refused, before its CUDA call is made
  static bool refused() {
    int64_t n = g_refuse_after.load();
    while (n >= 0 && !g_refuse_after.compare_exchange_weak(n, n - 1)) {
    }
    return n == 0;
  }
  // one acquisition's result (`e`, its CUDA call's or its refusal's): recorded and handed to `out` if it succeeded
  template <typename P>
  int keep(cudaError_t e, const char* what, void* q, Kind kind, size_t bytes, cudaStream_t st, P& out) {
    if (e != cudaSuccess) return fail(PB_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
    held.push_back({q, kind, bytes, st, -1, 0, 0});
    g_owned_count += 1;
    g_owned_bytes += bytes;
    out = static_cast<P>(q);
    return PB_OK;
  }
  void drop(size_t i, cudaStream_t st) {
    const Res r = held[i];
    held.erase(held.begin() + i);
    switch (r.kind) {
      case DEV: cudaFree(r.p); break;
      case HOST: cudaFreeHost(r.p); break;
      case ASYNC: cudaFreeAsync(r.p, st); break;
      case STREAM: cudaStreamDestroy(static_cast<cudaStream_t>(r.p)); break;
      case EVENT: cudaEventDestroy(static_cast<cudaEvent_t>(r.p)); break;
      case IPC: cudaIpcCloseMemHandle(r.p); break;
      case SHARED:
        cudaHostUnregister(r.p);
        munmap(r.p, r.bytes);
        close(r.fd);
        break;
      case VRESERVE: vmm().free(reinterpret_cast<CUdeviceptr>(r.p), r.span); break;
      case VCHUNK:
        vmm().unmap(reinterpret_cast<CUdeviceptr>(r.p), r.bytes);
        vmm().release((CUmemGenericAllocationHandle)r.handle);
        break;
    }
    g_owned_count -= 1;
    g_owned_bytes -= r.bytes;
  }
};

}  // namespace
