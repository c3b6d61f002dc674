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
inline bool ensure_func_attribute(Kernel kernel, cudaFuncAttribute attr, int value, std::atomic<unsigned long long>* done_mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  const unsigned long long bit = 1ull << (dev & 63);
  if (done_mask->load(std::memory_order_acquire) & bit) return true;
  if (cudaFuncSetAttribute(kernel, attr, value) != cudaSuccess) return false;
  done_mask->fetch_or(bit, std::memory_order_release);
  return true;
}

template <typename Kernel>
inline bool ensure_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>* done_mask) {
  return ensure_func_attribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes, done_mask);
}

// The same launch with the CTAs grouped into thread-block clusters of `cluster` (no cluster attribute when it is 1 x 1 x 1).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 cluster, dim3 block, size_t smem,
                                      cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster.x * cluster.y * cluster.z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster.x;
    attr[n].val.clusterDim.y = cluster.y;
    attr[n].val.clusterDim.z = cluster.z;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  return launch_pdl_cluster(kernel, grid, dim3(1, 1, 1), block, smem, st, static_cast<Args&&>(args)...);
}

}  // namespace b200
