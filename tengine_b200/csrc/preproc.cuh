// preproc.cuh -- what the input preprocessing kernels (image_pre.cu, detect_pre.cu) share: the examples' float -> int conversion.
#pragma once
#include <climits>

namespace tb200 {

// round(x) of <math.h> (halfway cases away from zero), then the conversion to int of the x86-64 build: a value outside int's range,
// or NaN, becomes INT_MIN (cvttsd2si), which the examples' clamps then send to their lower bound.
__device__ __forceinline__ int round_to_int_x86(float x)
{
    float r = truncf(x);
    if (fabsf(__fsub_rn(x, r)) >= 0.5f) r = __fadd_rn(r, copysignf(1.f, x));
    return (r >= -2147483648.f && r < 2147483648.f) ? (int)r : INT_MIN;
}

} // namespace tb200
