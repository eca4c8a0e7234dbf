// fast_api.h -- host entry points of the specialised streaming kernels; each is defined in its own translation
// unit (k_afb.cu, k_sfb.cu, k_dtcwt_fwd.cu, k_dtcwt_inv.cu, k_pyramid.cu) so the library builds in parallel.
// Every function returns 0 when it launched, kNoFastPath when there is no specialisation for these parameters
// (the caller then runs the generic tile kernel), or a negative B200W_E* code.  No global state.
#pragma once
#include <cuda_runtime.h>

#include "common.h"
#include "dtcwt_fwd12_plan.h"
#include "pyramid_plan.h"

namespace b200w {
namespace fast {

constexpr int kNoFastPath = 1;

int try_launch_afb(const AfbParams& p, cudaStream_t stream);
int try_launch_sfb(const SfbParams& p, cudaStream_t stream);
// the same levels on the wavelet-packet layout (children 4p .. 4p+3 of plane p; see wpt2d.cu)
int try_launch_wpt_afb(const AfbParams& p, cudaStream_t stream);
int try_launch_wpt_sfb(const SfbParams& p, cudaStream_t stream);
int try_launch_fwd_j1(const DtParams& p, cudaStream_t stream);
int try_launch_scat_j1(const DtParams& p, cudaStream_t stream);
int try_launch_fwd_j2plus(const DtParams& p, cudaStream_t stream);
int try_launch_inv_j1(const DtParams& p, cudaStream_t stream);
int try_launch_inv_j2plus(const DtParams& p, cudaStream_t stream);
// DTCWT forward levels 1 and 2 in one kernel (k_dtcwt_fwd.cu): p1 = level 1 (its `out` unused), p2 = level 2 (its `in`
// unused); kNoFastPath unless fwd12_route accepts the call
int try_launch_fwd12(const DtParams& p1, const DtParams& p2, cudaStream_t stream);

// fused multi-level DWT analysis (k_pyramid.cu): plan_dwt_pyramid fills everything but the output pointers and the
// taps and returns kNoFastPath when the fused kernel does not apply (then run the levels one by one)
// (ll_pitch: row pitch of the final low-pass the kernel writes, 0 = contiguous)
int plan_dwt_pyramid(PyrParams& p, const float* x, long long xps, int xpitch, int planes, int H, int W, int J, int L,
                     int mode, int ll_pitch);
int launch_dwt_pyramid(const PyrParams& p, cudaStream_t stream);

}  // namespace fast
}  // namespace b200w
