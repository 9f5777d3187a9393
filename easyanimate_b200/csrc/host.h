// Host-side helpers shared by the C-ABI translation units: error reporting, kernel launch, TMA descriptor encoding
// (cuTensorMapEncodeTiled looked up through the runtime so the library has no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/ea_b200.h"

namespace ea {

int fail(int code, const std::string& msg);
int check_launch(const char* what);

// 2-D..5-D bf16 tiled tensor map. dims[0] is the contiguous dimension. strides_bytes has rank-1 entries
// (stride of dims[1..]). swizzle128: box inner extent must be 64 bf16 (128 B).
// elem_strides (optional, rank entries): traversal stride per dimension (the box then spans box[i] ELEMENTS OF THE TENSOR and
// ceil(box[i] / elem_strides[i]) of them are loaded).
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, bool swizzle128, const uint32_t* elem_strides = nullptr);

int sm_count();  // of the CURRENT device (cached per device)
int current_device();

// "done once" state that is per DEVICE: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) applies to the current device
// only, so a process that drives a second GPU (module.to("cuda:1") after work on cuda:0) must set it there too.
struct PerDeviceFlag {
  bool done[64] = {};
  bool get(int dev) const { return dev >= 0 && dev < 64 && done[dev]; }
  void set(int dev) {
    if (dev >= 0 && dev < 64) done[dev] = true;
  }
};

void count_launch();

// Raises kern's dynamic shared-memory limit to `bytes` on the current device, once per device (`done` belongs to kern).
int set_max_dynamic_smem(const void* kern, int bytes, PerDeviceFlag& done, const char* what);

// Blocks of `threads` needed to cover n work items.
inline unsigned grid_1d(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// Launches kern(args...) on `stream` (the C ABI's void* stream), counts the launch for ea_launch_count() and reports a
// launch error under the name `what`. Every kernel launch of the library goes through here.
template <class... Params, class... Args>
int launch(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem_bytes, void* stream, const char* what,
           const Args&... args) {
  kern<<<grid, block, smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(args...);
  count_launch();
  return check_launch(what);
}

// launch() as a persistent grid of min(tiles, SMs) CTAs of `threads` with `smem_bytes` of dynamic shared memory
// (set_max_dynamic_smem with `smem_done` first).
template <class... Params, class... Args>
int launch_persistent(void (*kern)(Params...), int64_t tiles, int threads, int smem_bytes, PerDeviceFlag& smem_done,
                      void* stream, const char* what, const Args&... args) {
  const int rc = set_max_dynamic_smem(reinterpret_cast<const void*>(kern), smem_bytes, smem_done, what);
  if (rc) return rc;
  return launch(kern, (unsigned)(tiles < sm_count() ? tiles : sm_count()), threads, smem_bytes, stream, what, args...);
}

}  // namespace ea

#define EA_REQUIRE(cond, msg)                                   \
  do {                                                          \
    if (!(cond)) return ::ea::fail(EA_ERR_INVALID, msg);  \
  } while (0)
