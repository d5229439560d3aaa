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
    for (int64_t e = tid; e < (int64_t)m * n; e += T) A[e] = A_in[b.a_off + e];
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
    for (int64_t e = tid; e < (int64_t)k * n; e += T) R_out[b.r_off + e] = A[e];
}

static inline int64_t qr_work_elems(int64_t m, int64_t n) {
    const int64_t k = std::min(m, n);
    int64_t w = m * n + m * k + 2 * k;
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
