// k_afb.cu -- translation unit of afb_stream.cuh (sm_90a): the DWT-layout analysis kernels
#include "afb_stream.cuh"

namespace b200w {
namespace fast {
int try_launch_afb(const AfbParams& p, cudaStream_t stream) { return try_launch_afb_layout<false>(p, stream); }
}  // namespace fast
}  // namespace b200w
