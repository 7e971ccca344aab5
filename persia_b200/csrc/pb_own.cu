// pb_own.cu — the one definition of the C ABI's error state, its resource counters and refusals, the driver's
// virtual-memory calls, and the parts of Owned that are not templates (pb_own.cuh).
#include <type_traits>

#include "pb_own.cuh"

namespace pb {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

std::atomic<uint64_t> g_owned_count{0}, g_owned_bytes{0};
std::atomic<int64_t> g_refuse_after{-1};

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
    w.share = w.ok & get("cuMemExportToShareableHandle", w.export_fd) & get("cuMemImportFromShareableHandle", w.import_fd) &
              get("cuDeviceGet", w.device_get) & get("cuDeviceGetAttribute", w.attribute);
    return w;
  }();
  return v;
}

namespace {
CUmemAllocationProp vmm_prop(int device, bool shareable = false) {
  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  if (shareable) prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return prop;
}
}  // namespace

size_t vmm_granularity(int device) {
  const Vmm& v = vmm();
  size_t g = 0;
  const CUmemAllocationProp prop = vmm_prop(device);
  if (!v.ok || v.granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS) return 0;
  return g;
}

bool vmm_fd_supported(int device) {
  const Vmm& v = vmm();
  CUdevice d = 0;
  int on = 0;
  if (!v.share || v.device_get(&d, device) != CUDA_SUCCESS ||
      v.attribute(&on, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, d) != CUDA_SUCCESS)
    return false;
  return on != 0;
}

Owned::~Owned() {
  while (!held.empty()) drop(held.size() - 1, held.back().st);
}

int Owned::stream(cudaStream_t& s) {
  cudaStream_t q = nullptr;
  const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking);
  return keep(e, "cudaStreamCreateWithFlags", q, STREAM, 0, nullptr, s);
}

int Owned::event(cudaEvent_t& ev) {
  cudaEvent_t q = nullptr;
  const cudaError_t e = refused() ? cudaErrorMemoryAllocation : cudaEventCreateWithFlags(&q, cudaEventDisableTiming);
  return keep(e, "cudaEventCreateWithFlags", q, EVENT, 0, nullptr, ev);
}

int Owned::chunk(void* at, size_t bytes, int device, bool shareable, unsigned long long* handle) {
  const Vmm& v = vmm();
  const CUmemAllocationProp prop = vmm_prop(device, shareable);
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
  if (handle) *handle = (unsigned long long)h;
  return PB_OK;
}

int Owned::import_chunk(void* at, size_t bytes, int fd, int device) {
  const Vmm& v = vmm();
  CUmemGenericAllocationHandle h = 0;
  if (refused()) {
    close(fd);
    return fail(PB_ERR_CUDA, "cuMemImportFromShareableHandle: refused");
  }
  CUresult e = v.import_fd(&h, reinterpret_cast<void*>((uintptr_t)fd), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  close(fd);  // (the handle holds the allocation from here on)
  if (e != CUDA_SUCCESS) return fail(PB_ERR_CUDA, "cuMemImportFromShareableHandle: CUresult " + std::to_string((int)e));
  const CUdeviceptr q = reinterpret_cast<CUdeviceptr>(at);
  if ((e = v.map(q, bytes, 0, h, 0)) == CUDA_SUCCESS) {
    CUmemAccessDesc acc;
    std::memset(&acc, 0, sizeof(acc));
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READ;  // a reader never writes the owner's rows or cells ...
    if (v.access(q, bytes, &acc, 1) != CUDA_SUCCESS) {
      acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;  // ... where the driver can map device memory read-only
      if ((e = v.access(q, bytes, &acc, 1)) != CUDA_SUCCESS) v.unmap(q, bytes);
    }
  }
  if (e != CUDA_SUCCESS) {
    v.release(h);
    return fail(PB_ERR_CUDA, "cuMemMap / cuMemSetAccess of an imported chunk: CUresult " + std::to_string((int)e));
  }
  held.push_back({at, VCHUNK, bytes, nullptr, -1, 0, (unsigned long long)h});
  g_owned_count += 1;
  g_owned_bytes += bytes;
  return PB_OK;
}

int Owned::ipc(void*& p, const cudaIpcMemHandle_t& h) {
  void* q = nullptr;
  const cudaError_t e =
      refused() ? cudaErrorMapBufferObjectFailed : cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
  return keep(e, "cudaIpcOpenMemHandle", q, IPC, 0, nullptr, p);
}

void Owned::release_all(cudaStream_t st) {
  while (!held.empty()) drop(held.size() - 1, st);
}

void Owned::adopt(Owned& o) {
  held.insert(held.end(), o.held.begin(), o.held.end());
  o.held.clear();
}

bool Owned::refused() {
  int64_t n = g_refuse_after.load();
  while (n >= 0 && !g_refuse_after.compare_exchange_weak(n, n - 1)) {
  }
  return n == 0;
}

void Owned::drop(size_t i, cudaStream_t st) {
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

}  // namespace pb
