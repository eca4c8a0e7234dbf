// k_wpt_stream.cu -- the streaming analysis / synthesis kernels compiled for the wavelet-packet layout (sm_90a), used by
// wpt2d.cu.  A translation unit of their own, so k_afb.cu / k_sfb.cu instantiate exactly the DWT kernels they always
// did and those compile to the same code.
#include "afb_stream.cuh"
#include "sfb_stream.cuh"

namespace b200w {
namespace fast {
int try_launch_wpt_afb(const AfbParams& p, cudaStream_t stream) { return try_launch_afb_layout<true>(p, stream); }
int try_launch_wpt_sfb(const SfbParams& p, cudaStream_t stream) { return try_launch_sfb_layout<true>(p, stream); }
}  // namespace fast
}  // namespace b200w
