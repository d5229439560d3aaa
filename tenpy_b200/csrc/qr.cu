// qr.cu -- batched Householder QR of the charge blocks of a matrix: one CTA per block, one launch per Array.
//
// Replaces the per-block LAPACK call of the reference's npc.qr (tenpy/linalg/np_conserved.py:4139, `np.linalg.qr`).
// Algorithm and phase functions: block_qr_core.cuh (host-checked, real and complex, by tests/csrc/block_qr_host.cpp;
// checked on the GPU against LAPACK at edge shapes by tests/test_gpu_kernel_edges.py).  One kernel, instantiated for real
// blocks (b200_block_qr_f64) and planar complex blocks (b200_block_qr_z).  npc.qr sends every real block of at most 384
// rows and columns here (np_conserved.QR_HOUSEHOLDER_MAX), larger real blocks to a Gram-Schmidt composition of the GEMM /
// BLAS-1 kernels, and complex blocks of every size here.
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

// CPLX: the imaginary planes Ai_in / Qi_out / Ri_out are used (planar complex blocks); otherwise they are ignored
template <bool CPLX>
__global__ void __launch_bounds__(QR_THREADS) block_qr_kernel(const QrBlk *__restrict__ blks,
                                                              const double *__restrict__ A_in, const double *__restrict__ Ai_in,
                                                              double *__restrict__ Q_out, double *__restrict__ Qi_out,
                                                              double *__restrict__ R_out, double *__restrict__ Ri_out,
                                                              double *__restrict__ work) {
    constexpr int P = CPLX ? 2 : 1;                   // planes
    __shared__ double partial[QR_THREADS];
    __shared__ double params[5];                      // bqr::reflector: Re tau, Re scale, beta, Im tau, Im scale
    const QrBlk b = blks[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x;
    const int m = b.m, n = b.n, k = b.k;
    const int64_t mn = (int64_t)m * n, mk = (int64_t)m * k;
    double *A = work + b.w_off, *Ai = CPLX ? A + mn : nullptr;   // m x n working copy, becomes R in its first k rows
    double *V = A + P * mn, *Vi = CPLX ? V + mk : nullptr;       // m x k reflectors
    double *tau = V + P * mk, *taui = CPLX ? tau + k : nullptr;  // k
    double *sign = tau + P * k;                                  // k
    const double *a_in = A_in + b.a_off, *ai_in = CPLX ? Ai_in + b.a_off : nullptr;
    double *Q = Q_out + b.q_off, *Qi = CPLX ? Qi_out + b.q_off : nullptr;
    bqr::absmax_partial(tid, T, a_in, ai_in, mn, partial);
    __syncthreads();
    const double scale = bqr::block_scale(T, partial), rscale = 1.0 / scale;   // exact: powers of two
    bqr::scale_in(tid, T, a_in, A, mn, scale, ai_in, Ai);
    __syncthreads();
    for (int j = 0; j < k; ++j) {
        bqr::col_partial(tid, T, A, m, n, j, partial, Ai);
        __syncthreads();
        if (tid == 0) {
            bqr::reflector(T, A, n, j, partial, params, Ai);
            tau[j] = params[0];
            if (CPLX) taui[j] = params[3];
        }
        __syncthreads();
        bqr::store_reflector(tid, T, A, V, m, n, k, j, params, Ai, Vi);
        __syncthreads();
        bqr::apply_reflector(tid, T, A, n, V, m, k, j, j + 1, params[0], Ai, Vi, CPLX ? -params[3] : 0.0);   // H^H A
        __syncthreads();
    }
    bqr::init_q(tid, T, Q, m, k, Qi);
    __syncthreads();
    for (int j = k - 1; j >= 0; --j) {
        bqr::apply_reflector(tid, T, Q, k, V, m, k, j, j, tau[j], Qi, Vi, CPLX ? taui[j] : 0.0);
        __syncthreads();
    }
    bqr::sign_of_diag(tid, T, A, n, k, sign);
    __syncthreads();
    bqr::flip_signs(tid, T, A, Q, m, n, k, sign, Ai, Qi);
    __syncthreads();
    bqr::store_r(tid, T, A, R_out + b.r_off, k, n, rscale, Ai, CPLX ? Ri_out + b.r_off : nullptr);
}

// scratch of one block: A and V (and tau) per plane, sign
static inline int64_t qr_work_elems(int64_t m, int64_t n, bool cplx) {
    const int64_t k = std::min(m, n);
    const int64_t w = (cplx ? 2 : 1) * (m * n + m * k + k) + k;
    return (w + 15) / 16 * 16;
}

static int64_t qr_worksize(int64_t nblocks, const int64_t *m, const int64_t *n, bool cplx) {
    int64_t elems = 0;
    for (int64_t i = 0; i < nblocks; ++i) elems += qr_work_elems(m[i], n[i], cplx);
    return elems * (int64_t)sizeof(double) + ((nblocks * (int64_t)sizeof(QrBlk) + 255) / 256 * 256);
}

// real (Ai == NULL) and complex (planar: A + i Ai -> Q + i Qi, R + i Ri) block QR: one host driver
static int block_qr_impl(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off, const int64_t *q_off,
                         const int64_t *r_off, const double *A, const double *Ai, double *Q, double *Qi, double *R,
                         double *Ri, void *work, int64_t work_bytes, b200_stream_t stream) {
    if (nblocks <= 0) return B200_OK;
    const bool cplx = Ai != nullptr;
    if (nblocks > 2147483647) return set_error(B200_ERR_ARG, "block_qr: too many blocks");
    if (work_bytes < qr_worksize(nblocks, m, n, cplx)) return set_error(B200_ERR_ARG, "block_qr: work buffer too small");
    std::vector<QrBlk> blks((size_t)nblocks);
    int64_t at = 0;
    for (int64_t i = 0; i < nblocks; ++i) {
        if (m[i] <= 0 || n[i] <= 0 || m[i] > 2147483647 || n[i] > 2147483647)
            return set_error(B200_ERR_ARG, "block_qr: bad block shape");
        blks[(size_t)i] = QrBlk{a_off[i], q_off[i], r_off[i], at, (int32_t)m[i], (int32_t)n[i],
                                (int32_t)std::min(m[i], n[i]), 0};
        at += qr_work_elems(m[i], n[i], cplx);
    }
    char *w = static_cast<char *>(work);
    QrBlk *d_blks = reinterpret_cast<QrBlk *>(w + at * (int64_t)sizeof(double));
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA_CHECK(cudaMemcpyAsync(d_blks, blks.data(), blks.size() * sizeof(QrBlk), cudaMemcpyHostToDevice, st));
    if (cplx)
        block_qr_kernel<true><<<(unsigned)nblocks, QR_THREADS, 0, st>>>(d_blks, A, Ai, Q, Qi, R, Ri,
                                                                        reinterpret_cast<double *>(w));
    else
        block_qr_kernel<false><<<(unsigned)nblocks, QR_THREADS, 0, st>>>(d_blks, A, nullptr, Q, nullptr, R, nullptr,
                                                                         reinterpret_cast<double *>(w));
    B200_CHECK_LAUNCH();
    B200_CUDA_CHECK(cudaStreamSynchronize(st));       // `blks` (pageable host memory) must outlive the copy
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_block_qr_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    return qr_worksize(nblocks, m, n, false);
}

extern "C" int b200_block_qr_f64(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                                 const int64_t *q_off, const int64_t *r_off, const double *A, double *Q, double *R,
                                 void *work, int64_t work_bytes, b200_stream_t stream) {
    return block_qr_impl(nblocks, m, n, a_off, q_off, r_off, A, nullptr, Q, nullptr, R, nullptr, work, work_bytes, stream);
}

extern "C" int64_t b200_block_qr_z_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    return qr_worksize(nblocks, m, n, true);
}

extern "C" int b200_block_qr_z(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                               const int64_t *q_off, const int64_t *r_off, const double *A_re, const double *A_im,
                               double *Q_re, double *Q_im, double *R_re, double *R_im, void *work, int64_t work_bytes,
                               b200_stream_t stream) {
    if (nblocks > 0 && (A_re == nullptr || A_im == nullptr))
        return set_error(B200_ERR_ARG, "complex QR: both planes of A are needed");
    return block_qr_impl(nblocks, m, n, a_off, q_off, r_off, A_re, A_im, Q_re, Q_im, R_re, R_im, work, work_bytes, stream);
}
