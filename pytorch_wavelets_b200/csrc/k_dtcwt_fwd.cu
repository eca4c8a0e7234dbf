// k_dtcwt_fwd.cu -- translation unit of dtcwt_fwd_stream.cuh and dtcwt_fwd12.cuh (sm_90a)
#include "dtcwt_fwd_stream.cuh"
#include "dtcwt_fwd12.cuh"
