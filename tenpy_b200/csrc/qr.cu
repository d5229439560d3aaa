// qr.cu -- batched Householder QR of the charge blocks of a matrix: one CTA per block, one launch per Array.
//
// Replaces the per-block LAPACK call of the reference's npc.qr (tenpy/linalg/np_conserved.py:4139, `np.linalg.qr`).
// Algorithm and phase functions: block_qr_core.cuh (host-checked by tests/csrc/block_qr_host.cpp; checked on the GPU
// against LAPACK at edge shapes by tests/test_gpu_kernel_edges.py).  npc.qr uses it for every block of at most 384 rows and
// columns (np_conserved.qr_method = 'auto', the default; 'householder' sends every block here); larger blocks go to a
// Gram-Schmidt composition of the GEMM / BLAS-1 kernels.
#include <algorithm>
#include <vector>

#include "block_qr_core.cuh"
#include "common.cuh"

namespace b200 {

constexpr int QR_THREADS = 256;

struct QrBlk {
    int64_t a_off, q_off, r_off, w_off;   // element offsets: A / Q / R in the caller's buffers, scratch in `work`
    int32_t m, n, k, pad;
};

__global__ void __launch_bounds__(QR_THREADS) block_qr_kernel(const QrBlk *__restrict__ blks,
                                                              const double *__restrict__ A_in, double *__restrict__ Q_out,
                                                              double *__restrict__ R_out, double *__restrict__ work) {
    __shared__ double partial[QR_THREADS];
    __shared__ double params[3];
    const QrBlk b = blks[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x;
    const int m = b.m, n = b.n, k = b.k;
    double *A = work + b.w_off;                       // m x n working copy, becomes R in its first k rows
    double *V = A + (int64_t)m * n;                   // m x k reflectors
    double *tau = V + (int64_t)m * k;                 // k
    double *sign = tau + k;                           // k
    double *Q = Q_out + b.q_off;
    bqr::absmax_partial(tid, T, A_in + b.a_off, nullptr, (int64_t)m * n, partial);
    __syncthreads();
    const double scale = bqr::block_scale(T, partial), rscale = 1.0 / scale;   // exact: powers of two
    bqr::scale_in(tid, T, A_in + b.a_off, A, (int64_t)m * n, scale);
    __syncthreads();
    for (int j = 0; j < k; ++j) {
        bqr::col_partial(tid, T, A, m, n, j, partial);
        __syncthreads();
        if (tid == 0) {
            bqr::reflector(T, A, n, j, partial, params);
            tau[j] = params[0];
        }
        __syncthreads();
        bqr::store_reflector(tid, T, A, V, m, n, k, j, params);
        __syncthreads();
        bqr::apply_reflector(tid, T, A, n, V, m, k, j, j + 1, params[0]);
        __syncthreads();
    }
    bqr::init_q(tid, T, Q, m, k);
    __syncthreads();
    for (int j = k - 1; j >= 0; --j) {
        bqr::apply_reflector(tid, T, Q, k, V, m, k, j, j, tau[j]);
        __syncthreads();
    }
    bqr::sign_of_diag(tid, T, A, n, k, sign);
    __syncthreads();
    bqr::flip_signs(tid, T, A, Q, m, n, k, sign);
    __syncthreads();
    bqr::store_r(tid, T, A, R_out + b.r_off, k, n, rscale);
}

static inline int64_t qr_work_elems(int64_t m, int64_t n) {
    const int64_t k = std::min(m, n);
    int64_t w = m * n + m * k + 2 * k;
    return (w + 15) / 16 * 16;
}

// ---- complex Householder QR (b200_block_qr_z): planar data, one CTA per block -----------------------------------------
// The unblocked zgeqr2 + zung2r pair: reflector j is H_j = 1 - tau_j v v^H with v[j] = 1 (zlarfg: beta real,
// |beta| = |column below and on the diagonal|), A <- H_j^H A for the columns right of j, Q = H_0 H_1 ... H_{k-1} applied to
// the first k columns of the identity.  R has a real diagonal by construction; rows of R / columns of Q with a negative
// diagonal entry change sign.  Threads own columns (coalesced rows); per-step partial sums are reduced in a fixed order.
__global__ void __launch_bounds__(QR_THREADS) block_qr_z_kernel(const QrBlk *__restrict__ blks, const double *__restrict__ Ar_in,
                                                                const double *__restrict__ Ai_in, double *__restrict__ Qr_out,
                                                                double *__restrict__ Qi_out, double *__restrict__ Rr_out,
                                                                double *__restrict__ Ri_out, double *__restrict__ work) {
    __shared__ double partial[QR_THREADS];
    __shared__ double params[5];                      // tau (re, im), scale (re, im), beta
    const QrBlk b = blks[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x;
    const int m = b.m, n = b.n, k = b.k;
    const int64_t mn = (int64_t)m * n, mk = (int64_t)m * k;
    double *Ar = work + b.w_off, *Ai = Ar + mn;       // m x n working copy, becomes R in its first k rows
    double *Vr = Ai + mn, *Vi = Vr + mk;              // m x k reflectors
    double *taur = Vi + mk, *taui = taur + k;         // k
    double *Qr = Qr_out + b.q_off, *Qi = Qi_out + b.q_off;
    bqr::absmax_partial(tid, T, Ar_in + b.a_off, Ai_in + b.a_off, mn, partial);
    __syncthreads();
    const double scale = bqr::block_scale(T, partial), rscale = 1.0 / scale;   // block_qr_core.cuh: exact
    for (int64_t e = tid; e < mn; e += T) {
        Ar[e] = Ar_in[b.a_off + e] * scale;
        Ai[e] = Ai_in[b.a_off + e] * scale;
    }
    __syncthreads();
    for (int j = 0; j < k; ++j) {
        double s = 0.0;
        for (int r = j + 1 + tid; r < m; r += T) {
            const double xr = Ar[(int64_t)r * n + j], xi = Ai[(int64_t)r * n + j];
            s = fma(xr, xr, fma(xi, xi, s));
        }
        partial[tid] = s;
        __syncthreads();
        if (tid == 0) {
            double sigma = 0.0;
            for (int t = 0; t < T; ++t) sigma += partial[t];
            const double ar = Ar[(int64_t)j * n + j], ai = Ai[(int64_t)j * n + j];
            if (sigma == 0.0 && ai == 0.0) {          // H = 1
                params[0] = params[1] = params[2] = params[3] = 0.0;
                params[4] = ar;
            } else {
                // beta = -sign(ar) |alpha, x|;  tau = (beta - alpha) / beta;  scale = 1 / (alpha - beta)
                const double nrm = sqrt(fma(ar, ar, fma(ai, ai, sigma)));
                const double beta = ar >= 0.0 ? -nrm : nrm;
                params[0] = (beta - ar) / beta;
                params[1] = -ai / beta;
                const double dr = ar - beta, di = ai, d2 = dr * dr + di * di;
                params[2] = dr / d2;
                params[3] = -di / d2;
                params[4] = beta;
            }
            taur[j] = params[0];
            taui[j] = params[1];
        }
        __syncthreads();
        const double scr = params[2], sci = params[3];
        for (int r = tid; r < m; r += T) {           // v = (0.., 1, x * scale); A[j][j] = beta, zeros below
            double vr = 0.0, vi = 0.0;
            const int64_t o = (int64_t)r * n + j;
            if (r == j) {
                vr = 1.0;
                Ar[o] = params[4];
                Ai[o] = 0.0;
            } else if (r > j) {
                vr = Ar[o] * scr - Ai[o] * sci;
                vi = Ar[o] * sci + Ai[o] * scr;
                Ar[o] = 0.0;
                Ai[o] = 0.0;
            }
            Vr[(int64_t)r * k + j] = vr;
            Vi[(int64_t)r * k + j] = vi;
        }
        __syncthreads();
        // A <- (1 - conj(tau) v v^H) A on the columns c > j:  w = v^H A[:, c],  A[:, c] -= conj(tau) w v
        const double tr = params[0], ti = -params[1];
        if (tr != 0.0 || ti != 0.0) {
            for (int c = j + 1 + tid; c < n; c += T) {
                double wr = 0.0, wi = 0.0;
                for (int r = j; r < m; ++r) {
                    const double vr = Vr[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
                    const double xr = Ar[(int64_t)r * n + c], xi = Ai[(int64_t)r * n + c];
                    wr = fma(vr, xr, fma(vi, xi, wr));
                    wi = fma(vr, xi, fma(-vi, xr, wi));
                }
                const double fr = tr * wr - ti * wi, fi = tr * wi + ti * wr;
                for (int r = j; r < m; ++r) {
                    const double vr = Vr[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
                    Ar[(int64_t)r * n + c] -= fr * vr - fi * vi;
                    Ai[(int64_t)r * n + c] -= fr * vi + fi * vr;
                }
            }
        }
        __syncthreads();
    }
    for (int64_t e = tid; e < mk; e += T) {
        Qr[e] = (e / k == e % k) ? 1.0 : 0.0;
        Qi[e] = 0.0;
    }
    __syncthreads();
    for (int j = k - 1; j >= 0; --j) {               // Q <- (1 - tau v v^H) Q on the columns c >= j
        const double tr = taur[j], ti = taui[j];
        if (tr != 0.0 || ti != 0.0) {
            for (int c = j + tid; c < k; c += T) {
                double wr = 0.0, wi = 0.0;
                for (int r = j; r < m; ++r) {
                    const double vr = Vr[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
                    const double xr = Qr[(int64_t)r * k + c], xi = Qi[(int64_t)r * k + c];
                    wr = fma(vr, xr, fma(vi, xi, wr));
                    wi = fma(vr, xi, fma(-vi, xr, wi));
                }
                const double fr = tr * wr - ti * wi, fi = tr * wi + ti * wr;
                for (int r = j; r < m; ++r) {
                    const double vr = Vr[(int64_t)r * k + j], vi = Vi[(int64_t)r * k + j];
                    Qr[(int64_t)r * k + c] -= fr * vr - fi * vi;
                    Qi[(int64_t)r * k + c] -= fr * vi + fi * vr;
                }
            }
        }
        __syncthreads();
    }
    // non-negative diagonal of R: the diagonal is real, flip the sign of row i of R and column i of Q where it is negative
    for (int64_t e = tid; e < (int64_t)k * n; e += T) {
        const int i = (int)(e / n), c = (int)(e % n);
        const double sg = Ar[(int64_t)i * n + i] < 0.0 ? -1.0 : 1.0;
        Rr_out[b.r_off + e] = c < i ? 0.0 : sg * Ar[e] * rscale;
        Ri_out[b.r_off + e] = c < i ? 0.0 : sg * Ai[e] * rscale;
    }
    for (int64_t e = tid; e < mk; e += T) {
        const int i = (int)(e % k);
        if (Ar[(int64_t)i * n + i] < 0.0) {
            Qr[e] = -Qr[e];
            Qi[e] = -Qi[e];
        }
    }
}

static inline int64_t qr_z_work_elems(int64_t m, int64_t n) {
    const int64_t k = std::min(m, n);
    int64_t w = 2 * (m * n + m * k + k);
    return (w + 15) / 16 * 16;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_block_qr_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    int64_t elems = 0;
    for (int64_t i = 0; i < nblocks; ++i) elems += qr_work_elems(m[i], n[i]);
    return elems * (int64_t)sizeof(double) + ((nblocks * (int64_t)sizeof(QrBlk) + 255) / 256 * 256);
}

extern "C" int b200_block_qr_f64(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                                 const int64_t *q_off, const int64_t *r_off, const double *A, double *Q, double *R,
                                 void *work, int64_t work_bytes, b200_stream_t stream) {
    if (nblocks <= 0) return B200_OK;
    if (work_bytes < b200_block_qr_worksize(nblocks, m, n)) return set_error(B200_ERR_ARG, "block_qr: work buffer too small");
    std::vector<QrBlk> blks((size_t)nblocks);
    int64_t at = 0;
    for (int64_t i = 0; i < nblocks; ++i) {
        if (m[i] <= 0 || n[i] <= 0 || m[i] > 2147483647 || n[i] > 2147483647)
            return set_error(B200_ERR_ARG, "block_qr: bad block shape");
        blks[(size_t)i] = QrBlk{a_off[i], q_off[i], r_off[i], at, (int32_t)m[i], (int32_t)n[i],
                                (int32_t)std::min(m[i], n[i]), 0};
        at += qr_work_elems(m[i], n[i]);
    }
    char *w = static_cast<char *>(work);
    QrBlk *d_blks = reinterpret_cast<QrBlk *>(w + at * (int64_t)sizeof(double));
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA_CHECK(cudaMemcpyAsync(d_blks, blks.data(), blks.size() * sizeof(QrBlk), cudaMemcpyHostToDevice, st));
    block_qr_kernel<<<(unsigned)nblocks, QR_THREADS, 0, st>>>(d_blks, A, Q, R, reinterpret_cast<double *>(w));
    B200_CHECK_LAUNCH();
    B200_CUDA_CHECK(cudaStreamSynchronize(st));       // `blks` (pageable host memory) must outlive the copy
    return B200_OK;
}

extern "C" int64_t b200_block_qr_z_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    int64_t elems = 0;
    for (int64_t i = 0; i < nblocks; ++i) elems += qr_z_work_elems(m[i], n[i]);
    return elems * (int64_t)sizeof(double) + ((nblocks * (int64_t)sizeof(QrBlk) + 255) / 256 * 256);
}

extern "C" int b200_block_qr_z(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                               const int64_t *q_off, const int64_t *r_off, const double *A_re, const double *A_im,
                               double *Q_re, double *Q_im, double *R_re, double *R_im, void *work, int64_t work_bytes,
                               b200_stream_t stream) {
    if (nblocks <= 0) return B200_OK;
    if (nblocks > 2147483647) return set_error(B200_ERR_ARG, "block_qr_z: too many blocks");
    if (work_bytes < b200_block_qr_z_worksize(nblocks, m, n)) return set_error(B200_ERR_ARG, "block_qr_z: work buffer too small");
    std::vector<QrBlk> blks((size_t)nblocks);
    int64_t at = 0;
    for (int64_t i = 0; i < nblocks; ++i) {
        if (m[i] <= 0 || n[i] <= 0 || m[i] > 2147483647 || n[i] > 2147483647)
            return set_error(B200_ERR_ARG, "block_qr_z: bad block shape");
        blks[(size_t)i] = QrBlk{a_off[i], q_off[i], r_off[i], at, (int32_t)m[i], (int32_t)n[i],
                                (int32_t)std::min(m[i], n[i]), 0};
        at += qr_z_work_elems(m[i], n[i]);
    }
    char *w = static_cast<char *>(work);
    QrBlk *d_blks = reinterpret_cast<QrBlk *>(w + at * (int64_t)sizeof(double));
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA_CHECK(cudaMemcpyAsync(d_blks, blks.data(), blks.size() * sizeof(QrBlk), cudaMemcpyHostToDevice, st));
    block_qr_z_kernel<<<(unsigned)nblocks, QR_THREADS, 0, st>>>(d_blks, A_re, A_im, Q_re, Q_im, R_re, R_im,
                                                                reinterpret_cast<double *>(w));
    B200_CHECK_LAUNCH();
    B200_CUDA_CHECK(cudaStreamSynchronize(st));       // `blks` (pageable host memory) must outlive the copy
    return B200_OK;
}
