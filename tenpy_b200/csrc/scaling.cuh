// scaling.cuh -- the power-of-two block scale of the decomposition kernels (host and device).
//
// The SVD, eigh and QR kernels form sums of squares (Gram entries, Householder norms) without per-element scaling.  They
// run on 2^-e A with 2^e the power of two of max |a_ij|, so that the largest entry lies in [1, 2) and these sums stay
// far from over- and underflow for any finite input.  Multiplication by a power of two is exact and commutes with every
// floating-point operation in the normal range: the scaled computation returns bit for bit the same vectors as the
// unscaled one wherever that one stays normal, and the values (S, R, W) scaled back by 2^e.
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif

namespace b200 {

// 2^-ilogb(amax), clamped to [2^-1022, 2^1022] so that the scale and its inverse are normal; 1 for a zero, inf or NaN amax
B200_HD double pow2_scale(double amax) {
    if (!(amax > 0.0) || !(amax <= 1.7976931348623157e308)) return 1.0;
    int e = -ilogb(amax);
    e = e < -1022 ? -1022 : (e > 1022 ? 1022 : e);
    return ldexp(1.0, e);
}

}  // namespace b200
