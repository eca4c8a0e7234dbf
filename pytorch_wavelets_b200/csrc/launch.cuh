// launch.cuh -- the one launch path of the generic tile kernels, the 1-D row kernels and the DTCWT primitives, and the
// error record behind b200w_last_cuda_error().
#pragma once
#include <cuda_runtime.h>

#include "../../include/b200wave.h"

namespace b200w {

// B200W_OK for cudaSuccess; otherwise records "<error name>: <error string>" in the calling thread's buffer that
// b200w_last_cuda_error() returns and gives B200W_ECUDA.  Defined in b200wave.cu.
int check_cuda(cudaError_t e);

inline int check_launch() { return check_cuda(cudaGetLastError()); }

// Launches kernel(p) on `blocks` CTAs of `threads` threads with `smem_bytes` of dynamic shared memory, opting in above
// the default 48 KB; more than an sm_90 CTA can have (227 KB) is B200W_EFILTER.  Nothing to do is B200W_OK.
template <class K, class P>
int launch(K kernel, const P& p, long long blocks, int threads, size_t smem_bytes, void* stream) {
  if (blocks == 0) return B200W_OK;
  if (smem_bytes > 48 * 1024) {
    if (smem_bytes > 227 * 1024) return B200W_EFILTER;
    const int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    if (rc) return rc;
  }
  kernel<<<(unsigned)blocks, threads, smem_bytes, (cudaStream_t)stream>>>(p);
  return check_launch();
}

}  // namespace b200w
