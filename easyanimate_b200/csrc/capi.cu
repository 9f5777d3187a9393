// Library-level entry points of the C ABI: error string, version, launch counter.
#include <atomic>
#include <string.h>

#include <string>

#include <cuda.h>

#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {
const char* last_error_cstr();
static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace ea

extern "C" const char* ea_last_error(void) { return ea::last_error_cstr(); }
extern "C" int ea_abi_version(void) { return 4; }
extern "C" uint64_t ea_launch_count(void) { return ea::g_launches.load(std::memory_order_relaxed); }

extern "C" int ea_enable_peer_access(int32_t peer_device) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return ea::fail(EA_ERR_CUDA, "ea_enable_peer_access: no current device");
  if (peer_device == dev) return EA_OK;
  int can = 0;
  cudaError_t e = cudaDeviceCanAccessPeer(&can, dev, peer_device);
  if (e != cudaSuccess || !can) {
    (void)cudaGetLastError();
    return ea::fail(EA_ERR_CUDA, "ea_enable_peer_access: device " + std::to_string(dev) + " cannot access device " + std::to_string(peer_device));
  }
  e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
    return ea::fail(EA_ERR_CUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
  (void)cudaGetLastError();
  return EA_OK;
}

// CUDA IPC import for the sequence-parallel peer buffers.  The mapping must be made with the IMPORTING kernel's device current
// (cudaIpcMemLazyEnablePeerAccess then sets up peer access from it to the exporting device): a mapping opened under the
// exporter's device index - what torch's own storage sharing does - is readable by copy engines but faults when a kernel
// of another device dereferences it.
// Export side: the 64-byte handle of the device allocation that contains `ptr` (cuMemGetAddressRange finds its base; torch's
// caching allocator sub-allocates from cudaMalloc'ed segments) and ptr's byte offset inside it.
extern "C" int ea_ipc_export(const void* ptr, void* handle64_out, int64_t* offset_out) {
  if (!ptr || !handle64_out || !offset_out) return ea::fail(EA_ERR_INVALID, "ea_ipc_export: null pointer");
  typedef CUresult (*GetRangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
  static GetRangeFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !f) {
      (void)cudaGetLastError();
      return ea::fail(EA_ERR_CUDA, "ea_ipc_export: cuMemGetAddressRange unavailable");
    }
    fn = reinterpret_cast<GetRangeFn>(f);
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  CUresult r = fn(&base, &size, reinterpret_cast<CUdeviceptr>(ptr));
  if (r != CUDA_SUCCESS) return ea::fail(EA_ERR_CUDA, "ea_ipc_export: cuMemGetAddressRange failed with CUresult " + std::to_string((int)r));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base));
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return ea::fail(EA_ERR_CUDA, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e) +
                                     " (the buffer must come from a cudaMalloc'ed segment: no expandable_segments / cudaMallocAsync)");
  }
  memcpy(handle64_out, &h, sizeof(h));
  *offset_out = (int64_t)(reinterpret_cast<CUdeviceptr>(ptr) - base);
  return EA_OK;
}

extern "C" int ea_ipc_open(const void* handle64, void** base_out) {
  if (!handle64 || !base_out) return ea::fail(EA_ERR_INVALID, "ea_ipc_open: null pointer");
  cudaIpcMemHandle_t h;
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(&h, handle64, sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return ea::fail(EA_ERR_CUDA, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
  }
  *base_out = p;
  return EA_OK;
}

extern "C" int ea_ipc_close(void* base) {
  if (!base) return EA_OK;
  cudaError_t e = cudaIpcCloseMemHandle(base);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return ea::fail(EA_ERR_CUDA, std::string("cudaIpcCloseMemHandle: ") + cudaGetErrorString(e));
  }
  return EA_OK;
}
