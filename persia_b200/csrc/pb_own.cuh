// pb_own.cuh — the C ABI's error reporting and the CUDA resources its objects hold (defined once, in pb_own.cu).
// Every buffer, mapped pinned host block, shared host mapping, stream-ordered buffer, stream, event and IPC mapping an
// object acquires is
// recorded in its Owned, which releases what is still held, in reverse order, when the object is deleted.  A step that
// acquires several resources acquires them into a local Owned and adopts it once every part has succeeded, then sets
// its gate: a step that fails leaves nothing allocated and no gate set, and the next call acquires afresh.
// A growable table's storage (pb_table_set_growth) is device address space reserved for its whole capacity and backed
// by physical memory chunk by chunk: the reservation and each chunk are resources of their own.  A view of an
// exportable growable table from another process reserves the same spans and maps the owner's chunks as they arrive.
#pragma once
#include <atomic>
#include <cerrno>
#include <cstring>
#include <string>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cuda.h>  // the driver's types only: its virtual-memory calls are reached through cudaGetDriverEntryPoint
#include <cuda_runtime.h>

#include "persia_b200.h"

namespace pb {

// the calling thread's last error message (pb_last_error)
extern thread_local std::string g_err;

int fail(int code, const std::string& msg);

#define PB_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return pb::fail(PB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));           \
  } while (0)

// what every live object holds (pb_debug_owned), and the acquisitions still granted before one is refused
// (pb_debug_refuse_after; -1: none is)
extern std::atomic<uint64_t> g_owned_count, g_owned_bytes;
extern std::atomic<int64_t> g_refuse_after;

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
  // exportable growth (pb_table_set_growth(t, 2)): chunks handed to other processes as POSIX file descriptors.  `share`
  // false: the driver lacks one of these (that mode is then refused; the others are unaffected)
  decltype(&cuMemExportToShareableHandle) export_fd = nullptr;
  decltype(&cuMemImportFromShareableHandle) import_fd = nullptr;
  decltype(&cuDeviceGet) device_get = nullptr;
  decltype(&cuDeviceGetAttribute) attribute = nullptr;
  bool share = false;
};

const Vmm& vmm();

// the size every chunk of `device` is a multiple of (0: no virtual-memory support)
size_t vmm_granularity(int device);
// whether `device` can export its chunks as POSIX file descriptors (CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED)
bool vmm_fd_supported(int device);

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
  ~Owned();

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
  int stream(cudaStream_t& s);
  int event(cudaEvent_t& ev);
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
  // reservation; undone as unmap, release.  shareable: created exportable as a POSIX file descriptor, its handle
  // written to `handle`
  int chunk(void* at, size_t bytes, int device, bool shareable = false, unsigned long long* handle = nullptr);
  // another process's chunk (`fd`, from cuMemExportToShareableHandle; closed here whatever happens), imported and
  // mapped at `at`, inside a reservation, for `device` to read (read-only where the driver allows it); undone as
  // unmap, release
  int import_chunk(void* at, size_t bytes, int fd, int device);
  // another process's allocation, mapped into this one
  int ipc(void*& p, const cudaIpcMemHandle_t& h);

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
  void release_all(cudaStream_t st);
  // take over what `o` holds (a step that has succeeded)
  void adopt(Owned& o);

 private:
  // pb_debug_refuse_after: this acquisition is refused, before its CUDA call is made
  static bool refused();
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
  void drop(size_t i, cudaStream_t st);
};

}  // namespace pb
