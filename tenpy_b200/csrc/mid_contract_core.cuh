// mid_contract_core.cuh -- OUT[o, n, i] = sum_k M[n, k] T[o, k, i]: a small matrix applied to the MIDDLE index of a
// 3-index tensor whose last index is contiguous.
//
// This is the step "apply the two-site MPO tensor W0.W1 to LP.theta" of the split-order effective-H matvec
// (algorithms/mps_common.py TwoSiteH._matvec_split): T = [vR*, (wL p0 p1), vR], M = [(p0' p1' wR), (wL p0 p1)],
// K = N = D d^2 (12 for the TFI chain).  Through npc.tensordot it costs two 100 MB block transpositions and a skinny
// GEMM; here T is read once and OUT written
// once, both coalesced along i, with no change of layout -- the output is exactly the operand the second large GEMM wants.
// One thread owns one (o, i) column: K loads (stride `inner`), N*K FMAs with M broadcast from shared memory, N stores.
//
// The per-thread body is a plain function shared with the host test (tests/csrc/mid_contract_host.cpp).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MC_HD __host__ __device__ __forceinline__
#else
#define MC_HD inline
#endif

namespace b200 {
namespace midc {

// column (o, i): t[k] = T[(o*K + k)*inner + i], OUT[(o*N + n)*inner + i] = sum_k M[n*K + k] t[k]
template <int KMAX>
MC_HD void column(int64_t o, int64_t i, int K, int N, int64_t inner, const double *M, const double *T, double *OUT) {
    double t[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) t[k] = (k < K) ? T[(o * K + k) * inner + i] : 0.0;
    for (int n = 0; n < N; ++n) {
        const double *m = M + (int64_t)n * K;
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) acc = fma(m[k], t[k], acc);
        OUT[(o * N + n) * inner + i] = acc;
    }
}

// two-segment version: the K index runs over T1 (K1 rows) then T2 (K2 rows), the N index over OUT1 (N1) then OUT2 (N2):
//   [OUT1; OUT2][o, n, i] = sum_k M[n, k] [T1; T2][o, k, i],   M: (N1 + N2) x (K1 + K2)
// This is the split-order matvec without the identity components of the environments (TwoSiteH._matvec_split_identity):
// T1 = LP_rest . theta, T2 = theta itself, OUT1 goes on to the contraction with RP_rest, OUT2 is added to the result.
template <int KMAX>
MC_HD void column2(int64_t o, int64_t i, int K1, int K2, int N1, int N2, int64_t inner, const double *M, const double *T1,
                   const double *T2, double *OUT1, double *OUT2) {
    const int K = K1 + K2;
    double t[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        double v = 0.0;
        if (k < K1)
            v = T1[(o * K1 + k) * inner + i];
        else if (k < K)
            v = T2[(o * K2 + (k - K1)) * inner + i];
        t[k] = v;
    }
    for (int n = 0; n < N1 + N2; ++n) {
        const double *m = M + (int64_t)n * K;
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) acc = fma(m[k], t[k], acc);
        if (n < N1)
            OUT1[(o * N1 + n) * inner + i] = acc;
        else
            OUT2[(o * N2 + (n - N1)) * inner + i] = acc;
    }
}

// complex two-segment version: M, T1, T2 complex, each stored planar (the real plane, then the imaginary plane of the
// same size: M at 0 and N*K, T1 at 0 and outer*K1*inner, T2 at 0 and outer*K2*inner).  OUT2 is planar as well.  OUT1
// is the left operand of the next GEMM (Y_rest . [RP_r; RP_i]) and is written as the real 2x2 embedding
// [[Yr, -Yi], [Yi, Yr]] of the matrix Y[(o, n / C1), (n % C1, i)] (rows m = outer*N1/C1, columns w = C1*inner; the
// embedding is 2m x 2w, row-major): every value of OUT1 is stored twice, so the GEMM needs no pass of its own.
template <int KMAX>
MC_HD void column2_z(int64_t o, int64_t i, int K1, int K2, int N1, int N2, int C1, int64_t outer, int64_t inner,
                     const double *Mr, const double *Mi, const double *T1, const double *T2, double *OUT1,
                     double *OUT2) {
    const int K = K1 + K2;
    const int64_t p1 = outer * K1 * inner, p2 = outer * K2 * inner;
    double tr[KMAX], ti[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        double vr = 0.0, vi = 0.0;
        if (k < K1) {
            const int64_t at = (o * K1 + k) * inner + i;
            vr = T1[at];
            vi = T1[p1 + at];
        } else if (k < K) {
            const int64_t at = (o * K2 + (k - K1)) * inner + i;
            vr = T2[at];
            vi = T2[p2 + at];
        }
        tr[k] = vr;
        ti[k] = vi;
    }
    const int P = N1 > 0 ? N1 / C1 : 0;
    const int64_t m = outer * P, w = (int64_t)C1 * inner, ld = 2 * w;
    const int64_t q2 = outer * N2 * inner;
    int pr = 0, pc = 0;                  // n = pr * C1 + pc while n < N1
    for (int n = 0; n < N1 + N2; ++n) {
        const double *mr = Mr + (int64_t)n * K, *mi = Mi + (int64_t)n * K;
        double ar = 0.0, ai = 0.0;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) {
                ar = fma(mr[k], tr[k], ar);
                ar = fma(-mi[k], ti[k], ar);
                ai = fma(mr[k], ti[k], ai);
                ai = fma(mi[k], tr[k], ai);
            }
        if (n < N1) {
            const int64_t row = o * P + pr, col = (int64_t)pc * inner + i;
            OUT1[row * ld + col] = ar;
            OUT1[row * ld + w + col] = -ai;
            OUT1[(m + row) * ld + col] = ai;
            OUT1[(m + row) * ld + w + col] = ar;
            if (++pc == C1) {
                pc = 0;
                ++pr;
            }
        } else {
            const int64_t at = (o * N2 + (n - N1)) * inner + i;
            OUT2[at] = ar;
            OUT2[q2 + at] = ai;
        }
    }
}

}  // namespace midc
}  // namespace b200
