// block_qr_core.cuh -- Householder QR of one row-major block, written as barrier-separated PHASES (one CTA per block).
//
// Replaces, per charge block, the LAPACK geqrf/orgqr pair behind the reference's npc.qr (np_conserved.py:4139,
// `np.linalg.qr(block, mode)`).  A (m x n, row-major) is overwritten by R (k x n upper triangular in its first k rows,
// k = min(m, n)), Q (m x k) is formed explicitly; the diagonal of R is made non-negative (the unique factorisation the
// reference returns for pos_diag_R=True).  Unblocked algorithm (dgeqr2 + dorg2r): right for the small and medium blocks of
// charge-conserving tensors, one launch per Array with no host round trip; big dense blocks want the blocked (compact WY)
// multi-CTA version -- round-2 work together with the QR preconditioning of the Jacobi SVD (DESIGN.md section 8).
//
// Complex blocks are planar: every phase takes the imaginary planes (Ai, Vi, Qi, ...) as trailing arguments, NULL (the
// default) for a real block.  The complex case is zgeqr2 + zung2r: reflector j is H_j = 1 - tau_j v v^H with v[j] = 1,
// complex tau and a real beta (zlarfg), A <- H_j^H A, Q = H_0 H_1 ... H_{k-1} applied to the first k columns of the
// identity; the diagonal of R is real by construction.  With the imaginary planes NULL every phase does exactly the real
// operations.
//
// Threads own COLUMNS (row-major storage: for a fixed row, consecutive threads touch consecutive addresses); the only
// cross-thread quantity per Householder step is the squared norm of the pivot column below the diagonal, summed in a
// fixed order from per-thread partials (deterministic).  Every phase is a plain function of (tid, nthreads, pointers):
// the CUDA kernel runs it per thread between __syncthreads(), tests/csrc/block_qr_host.cpp runs it for tid = 0..T-1.
//
// The factorisation runs on 2^-e A (scaling.cuh: the largest entry in [1, 2)), so that the column norms neither under- nor
// overflow for any finite block; R is scaled back exactly on output, Q is the same bit for bit.
#pragma once
#include <cmath>
#include <cstdint>

#include "scaling.cuh"

#if defined(__CUDACC__)
#define BQ_HD __host__ __device__ __forceinline__
#else
#define BQ_HD inline
#endif

namespace b200 {
namespace bqr {

// PHASE 0: partial[tid] = max |X[e]| over this thread's entries of the len entries of X (and Xi, if not NULL)
BQ_HD void absmax_partial(int tid, int T, const double *X, const double *Xi, int64_t len, double *partial) {
    double a = 0.0;
    for (int64_t e = tid; e < len; e += T) {
        a = fmax(a, fabs(X[e]));
        if (Xi) a = fmax(a, fabs(Xi[e]));
    }
    partial[tid] = a;
}

// PHASE 0 (every thread, after the barrier): the block scale pow2_scale(max |A|) from the partials
BQ_HD double block_scale(int T, const double *partial) {
    double a = 0.0;
    for (int t = 0; t < T; ++t) a = fmax(a, partial[t]);
    return b200::pow2_scale(a);
}

// PHASE 0 (after block_scale): A[e] = A_in[e] * scale (and Ai from Ai_in), the working copy the factorisation runs on
BQ_HD void scale_in(int tid, int T, const double *A_in, double *A, int64_t len, double scale,
                    const double *Ai_in = nullptr, double *Ai = nullptr) {
    for (int64_t e = tid; e < len; e += T) {
        A[e] = A_in[e] * scale;
        if (Ai) Ai[e] = Ai_in[e] * scale;
    }
}

// LAST PHASE: R_out = the first k rows of A times rscale = 1 / scale (exact: a power of two); Ri_out from Ai
BQ_HD void store_r(int tid, int T, const double *A, double *R_out, int k, int n, double rscale,
                   const double *Ai = nullptr, double *Ri_out = nullptr) {
    for (int64_t e = tid; e < (int64_t)k * n; e += T) {
        R_out[e] = A[e] * rscale;
        if (Ai) Ri_out[e] = Ai[e] * rscale;
    }
}

// PHASE 1: partial[tid] = sum over rows r > j (strided by threads) of |A[r][j]|^2
BQ_HD void col_partial(int tid, int T, const double *A, int m, int n, int j, double *partial,
                       const double *Ai = nullptr) {
    double s = 0.0;
    for (int r = j + 1 + tid; r < m; r += T) {
        const double a = A[(int64_t)r * n + j];
        if (Ai) {
            const double b = Ai[(int64_t)r * n + j];
            s = fma(a, a, fma(b, b, s));
        } else {
            s = fma(a, a, s);
        }
    }
    partial[tid] = s;
}

// A pivot column whose squared norm from the diagonal down is below this is negligible: the block is scaled so that
// max |a_ij| >= 2^-52, and the column is below 2^-450.  Its squares are subnormal or zero, so its norm would be
// inaccurate (a non-orthogonal reflector) or zero with alpha != 0 (tau and scale infinite).
constexpr double QR_NEGLIGIBLE_SQNORM = 0x1p-900;

// PHASE 2 (one thread): reflector H = 1 - tau v v^H with v[j] = 1 that maps the pivot column to beta e_j (H^H for a
// complex block), beta real: beta = -sign(Re alpha) |column from the diagonal down|, tau = (beta - alpha) / beta,
// scale = 1 / (alpha - beta).  params[0] = Re tau, params[1] = Re scale (v[r] = A[r][j] * scale for r > j),
// params[2] = beta; a complex block (Ai not NULL) also writes params[3] = Im tau, params[4] = Im scale.
// H = 1 (tau = scale = 0, beta = Re alpha) where the column below the diagonal and Im alpha are zero, and where the
// column is negligible (QR_NEGLIGIBLE_SQNORM): store_reflector then drops its entries below the diagonal and Im alpha,
// an absolute change below 2^-450 of a block whose largest entry is >= 2^-52.
BQ_HD void reflector(int T, const double *A, int n, int j, const double *partial, double *params,
                     const double *Ai = nullptr) {
    double sigma = 0.0;
    for (int t = 0; t < T; ++t) sigma += partial[t];
    const double alpha = A[(int64_t)j * n + j], ai = Ai ? Ai[(int64_t)j * n + j] : 0.0;
    if (Ai) params[3] = params[4] = 0.0;
    const double nrm2 = Ai ? fma(alpha, alpha, fma(ai, ai, sigma)) : alpha * alpha + sigma;
    if ((sigma == 0.0 && ai == 0.0) || nrm2 < QR_NEGLIGIBLE_SQNORM) {   // H = 1
        params[0] = 0.0;
        params[1] = 0.0;
        params[2] = alpha;
        return;
    }
    const double nrm = sqrt(nrm2);
    const double beta = alpha >= 0.0 ? -nrm : nrm;
    params[0] = (beta - alpha) / beta;
    if (Ai) {
        params[3] = -ai / beta;
        const double dr = alpha - beta, di = ai, d2 = dr * dr + di * di;
        params[1] = dr / d2;
        params[4] = -di / d2;
    } else {
        params[1] = 1.0 / (alpha - beta);
    }
    params[2] = beta;
}

// PHASE 3: store the reflector: V[r][j] = A[r][j] * scale (r > j), V[j][j] = 1, V[r][j] = 0 (r < j); A[r][j] = 0 below
// the diagonal, A[j][j] = beta.  V (and Vi) is m x k row-major.
BQ_HD void store_reflector(int tid, int T, double *A, double *V, int m, int n, int k, int j, const double *params,
                           double *Ai = nullptr, double *Vi = nullptr) {
    const double scr = params[1], sci = Ai ? params[4] : 0.0;
    for (int r = tid; r < m; r += T) {
        double vr = 0.0, vi = 0.0;
        if (r == j) {
            vr = 1.0;
            A[(int64_t)r * n + j] = params[2];
            if (Ai) Ai[(int64_t)r * n + j] = 0.0;
        } else if (r > j) {
            const int64_t o = (int64_t)r * n + j;
            if (Ai) {
                vr = A[o] * scr - Ai[o] * sci;
                vi = A[o] * sci + Ai[o] * scr;
                Ai[o] = 0.0;
            } else {
                vr = A[o] * scr;
            }
            A[o] = 0.0;
        }
        V[(int64_t)r * k + j] = vr;
        if (Vi) Vi[(int64_t)r * k + j] = vi;
    }
}

// PHASE 4: apply 1 - t v v^H (t = tau + i ti) to the columns c >= c0 of X (ld = ncol; X = A with t = conj(tau) and
// c0 = j + 1, or X = Q with t = tau and c0 = j): every thread owns columns c = c0 + tid, c0 + tid + T, ...:
// w = sum_{r >= j} conj(V[r][j]) X[r][c];  X[r][c] -= t w V[r][j]
BQ_HD void apply_reflector(int tid, int T, double *X, int ncol, const double *V, int m, int k, int j, int c0, double tau,
                           double *Xi = nullptr, const double *Vi = nullptr, double ti = 0.0) {
    if (tau == 0.0 && ti == 0.0) return;
    if (!Xi) {
        for (int c = c0 + tid; c < ncol; c += T) {
            double w = 0.0;
            for (int r = j; r < m; ++r) w = fma(V[(int64_t)r * k + j], X[(int64_t)r * ncol + c], w);
            w *= tau;
            for (int r = j; r < m; ++r) X[(int64_t)r * ncol + c] = fma(-V[(int64_t)r * k + j], w, X[(int64_t)r * ncol + c]);
        }
        return;
    }
    const double tr = tau;
    for (int c = c0 + tid; c < ncol; c += T) {
        double wr = 0.0, wi = 0.0;
        for (int r = j; r < m; ++r) {
            const double vr = V[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
            const double xr = X[(int64_t)r * ncol + c], xi = Xi[(int64_t)r * ncol + c];
            wr = fma(vr, xr, fma(vi, xi, wr));
            wi = fma(vr, xi, fma(-vi, xr, wi));
        }
        const double fr = tr * wr - ti * wi, fi = tr * wi + ti * wr;
        for (int r = j; r < m; ++r) {
            const double vr = V[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
            X[(int64_t)r * ncol + c] -= fr * vr - fi * vi;
            Xi[(int64_t)r * ncol + c] -= fr * vi + fi * vr;
        }
    }
}

// PHASE Q0: Q = first k columns of the identity
BQ_HD void init_q(int tid, int T, double *Q, int m, int k, double *Qi = nullptr) {
    for (int64_t e = tid; e < (int64_t)m * k; e += T) {
        Q[e] = (e / k == e % k) ? 1.0 : 0.0;
        if (Qi) Qi[e] = 0.0;
    }
}

// PHASE S: make diag(R) non-negative (it is real): rows i of R (= A) and columns i of Q with R[i][i] < 0 change sign.
// sign[i] must have been written by the previous phase (sign_of_diag).
BQ_HD void sign_of_diag(int tid, int T, const double *A, int n, int k, double *sign) {
    for (int i = tid; i < k; i += T) sign[i] = A[(int64_t)i * n + i] < 0.0 ? -1.0 : 1.0;
}
BQ_HD void flip_signs(int tid, int T, double *A, double *Q, int m, int n, int k, const double *sign,
                      double *Ai = nullptr, double *Qi = nullptr) {
    for (int64_t e = tid; e < (int64_t)k * n; e += T) {
        const int i = (int)(e / n);
        if (sign[i] < 0.0) {
            A[e] = -A[e];
            if (Ai) Ai[e] = -Ai[e];
        }
    }
    for (int64_t e = tid; e < (int64_t)m * k; e += T) {
        const int i = (int)(e % k);
        if (sign[i] < 0.0) {
            Q[e] = -Q[e];
            if (Qi) Qi[e] = -Qi[e];
        }
    }
}

}  // namespace bqr
}  // namespace b200
