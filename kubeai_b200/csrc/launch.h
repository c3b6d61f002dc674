// Kernel launch with the programmatic-stream-serialization attribute (PDL): the next kernel's
// prologue (and, for a decode-step GEMM, the weight loads of its first ring fill) overlaps the tail of the previous kernel.
// Every kernel launched this way executes griddepcontrol.wait before touching dependent memory.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <atomic>

namespace b200 {

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a kernel: one process may drive several GPUs
// (one engine per device), so "already set" is tracked per device ordinal.
template <typename Kernel>
inline bool ensure_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>* done_mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  const unsigned long long bit = 1ull << (dev & 63);
  if (done_mask->load(std::memory_order_acquire) & bit) return true;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return false;
  done_mask->fetch_or(bit, std::memory_order_release);
  return true;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200
