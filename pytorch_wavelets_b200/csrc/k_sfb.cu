// k_sfb.cu -- translation unit of sfb_stream.cuh (sm_90a): the DWT-layout synthesis kernels
#include "sfb_stream.cuh"

namespace b200w {
namespace fast {
int try_launch_sfb(const SfbParams& p, cudaStream_t stream) { return try_launch_sfb_layout<false>(p, stream); }
}  // namespace fast
}  // namespace b200w
