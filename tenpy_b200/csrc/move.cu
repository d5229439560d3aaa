// move.cu -- block data movement on packed block buffers (HBM-bandwidth bound): strided N-d block copies
// (transpose / combine_legs / split_legs), take-along-axis (iproject) and scale-along-axis (iscale_axis).
//
// Replaces the per-block numpy slicing of the reference: _sliced_copy (charges.py:1956 / pyx:754),
// Array_itranspose (pyx:813) + _imake_contiguous (pyx:1000), _combine_legs_worker (pyx:1013),
// _split_legs_worker (pyx:1136), Array.iproject (npc:1914), Array.iscale_axis (npc:2108).
// The integer "index plans" (records below) are computed on the host once per block layout and cached in
// device memory by the caller; a whole Array is moved by ONE launch.
#include "common.cuh"
#include "mid_contract_core.cuh"

namespace b200 {

constexpr int MV_THREADS = 256;

static inline dim3 mv_grid(int64_t n_tasks, int64_t max_elems, int per_thread) {
    int64_t chunks = (max_elems + (int64_t)MV_THREADS * per_thread - 1) / ((int64_t)MV_THREADS * per_thread);
    if (chunks < 1) chunks = 1;
    int64_t target = ((int64_t)sm_count() * 8 + n_tasks - 1) / n_tasks;
    if (target < 1) target = 1;
    int64_t gx = chunks < target ? chunks : target;
    return dim3((unsigned)gx, (unsigned)n_tasks);
}

// records: [soff, doff, n_elem, rank, shape[6], sstride[6], dstride[6]]
__global__ void __launch_bounds__(MV_THREADS) copy_blocks_kernel(const int64_t *__restrict__ tasks,
                                                                 const double *__restrict__ src,
                                                                 double *__restrict__ dst) {
    const int64_t *rec = tasks + (int64_t)blockIdx.y * B200_COPY_REC;
    const int64_t soff = rec[0], doff = rec[1], n = rec[2];
    const int rank = (int)rec[3];
    unsigned shape[B200_COPY_MAXRANK];
    int64_t ss[B200_COPY_MAXRANK], ds[B200_COPY_MAXRANK];
#pragma unroll
    for (int d = 0; d < B200_COPY_MAXRANK; ++d) {
        shape[d] = (unsigned)rec[4 + d];
        ss[d] = rec[4 + B200_COPY_MAXRANK + d];
        ds[d] = rec[4 + 2 * B200_COPY_MAXRANK + d];
    }
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        unsigned rem = (unsigned)e;  // n_elem < 2^32 is checked on the host
        int64_t so = soff, dd = doff;
#pragma unroll
        for (int d = B200_COPY_MAXRANK - 1; d >= 0; --d) {
            if (d < rank) {
                unsigned q = rem / shape[d];
                unsigned idx = rem - q * shape[d];
                rem = q;
                so += (int64_t)idx * ss[d];
                dd += (int64_t)idx * ds[d];
            }
        }
        dst[dd] = src[so];
    }
}

// records: [soff, doff, outer, n_keep, inner, src_len, idx_off]
__global__ void __launch_bounds__(MV_THREADS) take_blocks_kernel(const int64_t *__restrict__ tasks,
                                                                 const int64_t *__restrict__ idx,
                                                                 const double *__restrict__ src,
                                                                 double *__restrict__ dst) {
    const int64_t *rec = tasks + (int64_t)blockIdx.y * B200_TAKE_REC;
    const int64_t soff = rec[0], doff = rec[1], outer = rec[2], nk = rec[3], inner = rec[4], slen = rec[5],
                  ioff = rec[6];
    const int64_t n = outer * nk * inner;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        int64_t i = e % inner;
        int64_t r = e / inner;
        int64_t j = r % nk;
        int64_t o = r / nk;
        dst[doff + e] = src[soff + (o * slen + idx[ioff + j]) * inner + i];
    }
}

// records: [off, outer, len, inner, s_off]
__global__ void __launch_bounds__(MV_THREADS) scale_axis_kernel(const int64_t *__restrict__ tasks,
                                                                const double *__restrict__ s,
                                                                double *__restrict__ x) {
    const int64_t *rec = tasks + (int64_t)blockIdx.y * B200_SCALE_REC;
    const int64_t off = rec[0], outer = rec[1], len = rec[2], inner = rec[3], soff = rec[4];
    const int64_t n = outer * len * inner;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        int64_t j = (e / inner) % len;
        x[off + e] *= s[soff + j];
    }
}

// out[c] = sum_r X[r*ld + c]^2 : one thread per column, coalesced across the warp
__global__ void __launch_bounds__(MV_THREADS) col_sqnorms_kernel(int64_t rows, int64_t cols, int64_t ld,
                                                                 const double *__restrict__ x,
                                                                 double *__restrict__ out) {
    int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    double s = 0.0;
    for (int64_t r = 0; r < rows; ++r) {
        double v = x[r * ld + c];
        s = fma(v, v, s);
    }
    out[c] = s;
}

// OUT[o, n, i] = sum_k M[n, k] T[o, k, i]  (mid_contract_core.cuh); grid.x over i (256 per CTA), grid.y over o
template <int KMAX>
__global__ void __launch_bounds__(MV_THREADS) mid_contract_kernel(int K, int N, int64_t outer, int64_t inner,
                                                                  const double *__restrict__ M,
                                                                  const double *__restrict__ T,
                                                                  double *__restrict__ OUT) {
    extern __shared__ double sM[];
    for (int idx = threadIdx.x; idx < N * K; idx += blockDim.x) sM[idx] = M[idx];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= inner) return;
    for (int64_t o = blockIdx.y; o < outer; o += gridDim.y) midc::column<KMAX>(o, i, K, N, inner, sM, T, OUT);
}

template <int KMAX>
__global__ void __launch_bounds__(MV_THREADS) mid_contract2_kernel(int K1, int K2, int N1, int N2, int64_t outer,
                                                                   int64_t inner, const double *__restrict__ M,
                                                                   const double *__restrict__ T1,
                                                                   const double *__restrict__ T2,
                                                                   double *__restrict__ OUT1, double *__restrict__ OUT2) {
    extern __shared__ double sM[];
    for (int idx = threadIdx.x; idx < (N1 + N2) * (K1 + K2); idx += blockDim.x) sM[idx] = M[idx];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= inner) return;
    for (int64_t o = blockIdx.y; o < outer; o += gridDim.y)
        midc::column2<KMAX>(o, i, K1, K2, N1, N2, inner, sM, T1, T2, OUT1, OUT2);
}

// complex form (midc::column2_z): both planes of M in shared memory, one thread per (o, i) column
template <int KMAX>
__global__ void __launch_bounds__(MV_THREADS) mid_contract2_z_kernel(int K1, int K2, int N1, int N2, int C1,
                                                                     int64_t outer, int64_t inner,
                                                                     const double *__restrict__ M,
                                                                     const double *__restrict__ T1,
                                                                     const double *__restrict__ T2,
                                                                     double *__restrict__ OUT1,
                                                                     double *__restrict__ OUT2) {
    extern __shared__ double sM[];
    const int NK = (N1 + N2) * (K1 + K2);
    for (int idx = threadIdx.x; idx < 2 * NK; idx += blockDim.x) sM[idx] = M[idx];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= inner) return;
    for (int64_t o = blockIdx.y; o < outer; o += gridDim.y)
        midc::column2_z<KMAX>(o, i, K1, K2, N1, N2, C1, outer, inner, sM, sM + NK, T1, T2, OUT1, OUT2);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_mid_contract2_f64(int64_t K1, int64_t K2, int64_t N1, int64_t N2, int64_t outer, int64_t inner,
                                      const double *M_dev, const double *T1, const double *T2, double *OUT1, double *OUT2,
                                      b200_stream_t stream) {
    const int64_t K = K1 + K2, N = N1 + N2;
    if (outer <= 0 || inner <= 0 || N <= 0) return B200_OK;
    if (K1 < 0 || K2 < 0 || N1 < 0 || N2 < 0 || K <= 0 || K > 32 || N > 1024)
        return set_error(B200_ERR_ARG, "mid_contract2: K=%lld (1..32), N=%lld (<=1024)", (long long)K, (long long)N);
    const unsigned gx = (unsigned)((inner + MV_THREADS - 1) / MV_THREADS);
    const unsigned gy = (unsigned)(outer < 65535 ? outer : 65535);
    const size_t smem = (size_t)(N * K) * sizeof(double);
    if (smem > 48 * 1024) return set_error(B200_ERR_ARG, "mid_contract2: matrix %lld x %lld too large", (long long)N, (long long)K);
    if (K <= 16)
        mid_contract2_kernel<16><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K1, (int)K2, (int)N1, (int)N2, outer, inner, M_dev, T1, T2, OUT1, OUT2);
    else
        mid_contract2_kernel<32><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K1, (int)K2, (int)N1, (int)N2, outer, inner, M_dev, T1, T2, OUT1, OUT2);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_mid_contract2_z(int64_t K1, int64_t K2, int64_t N1, int64_t N2, int64_t C1, int64_t outer,
                                    int64_t inner, const double *M_dev, const double *T1, const double *T2, double *OUT1,
                                    double *OUT2, b200_stream_t stream) {
    const int64_t K = K1 + K2, N = N1 + N2;
    if (outer <= 0 || inner <= 0 || N <= 0) return B200_OK;
    if (K1 < 0 || K2 < 0 || N1 < 0 || N2 < 0 || K <= 0 || K > 32 || N > 1024)
        return set_error(B200_ERR_ARG, "mid_contract2_z: K=%lld (1..32), N=%lld (<=1024)", (long long)K, (long long)N);
    if (N1 > 0 && (C1 <= 0 || N1 % C1 != 0))
        return set_error(B200_ERR_ARG, "mid_contract2_z: C1=%lld does not divide N1=%lld", (long long)C1, (long long)N1);
    const unsigned gx = (unsigned)((inner + MV_THREADS - 1) / MV_THREADS);
    const unsigned gy = (unsigned)(outer < 65535 ? outer : 65535);
    const size_t smem = (size_t)(2 * N * K) * sizeof(double);
    if (smem > 48 * 1024)
        return set_error(B200_ERR_ARG, "mid_contract2_z: matrix %lld x %lld too large", (long long)N, (long long)K);
    const int c1 = N1 > 0 ? (int)C1 : 1;
    if (K <= 16)
        mid_contract2_z_kernel<16><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K1, (int)K2, (int)N1, (int)N2, c1, outer, inner, M_dev, T1, T2, OUT1, OUT2);
    else
        mid_contract2_z_kernel<32><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K1, (int)K2, (int)N1, (int)N2, c1, outer, inner, M_dev, T1, T2, OUT1, OUT2);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_mid_contract_f64(int64_t K, int64_t N, int64_t outer, int64_t inner, const double *M_dev,
                                     const double *T, double *OUT, b200_stream_t stream) {
    if (outer <= 0 || inner <= 0 || N <= 0) return B200_OK;
    if (K <= 0 || K > 32 || N > 1024) return set_error(B200_ERR_ARG, "mid_contract: K=%lld (1..32), N=%lld (<=1024)",
                                                        (long long)K, (long long)N);
    const unsigned gx = (unsigned)((inner + MV_THREADS - 1) / MV_THREADS);
    const unsigned gy = (unsigned)(outer < 65535 ? outer : 65535);
    const size_t smem = (size_t)(N * K) * sizeof(double);
    if (smem > 48 * 1024) return set_error(B200_ERR_ARG, "mid_contract: matrix %lld x %lld too large", (long long)N, (long long)K);
    if (K <= 16)
        mid_contract_kernel<16><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K, (int)N, outer, inner, M_dev, T, OUT);
    else
        mid_contract_kernel<32><<<dim3(gx, gy), MV_THREADS, smem, (cudaStream_t)stream>>>((int)K, (int)N, outer, inner, M_dev, T, OUT);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_col_sqnorms_f64(int64_t rows, int64_t cols, int64_t ld, const double *X, double *OUT,
                                    b200_stream_t stream) {
    if (cols <= 0) return B200_OK;
    col_sqnorms_kernel<<<(unsigned)((cols + MV_THREADS - 1) / MV_THREADS), MV_THREADS, 0, (cudaStream_t)stream>>>(
        rows, cols, ld, X, OUT);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_copy_blocks_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                                    const double *SRC, double *DST, b200_stream_t stream) {
    if (n_tasks <= 0) return B200_OK;
    if (n_tasks > 65535) return set_error(B200_ERR_ARG, "too many copy tasks (%lld)", (long long)n_tasks);
    int64_t max_n = 0;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t *rec = task_host + t * B200_COPY_REC;
        if (rec[3] < 0 || rec[3] > B200_COPY_MAXRANK) return set_error(B200_ERR_ARG, "copy task rank out of range");
        if (rec[2] >= (int64_t)1 << 32) return set_error(B200_ERR_ARG, "copy task too large");
        if (rec[2] > max_n) max_n = rec[2];
    }
    if (max_n == 0) return B200_OK;
    copy_blocks_kernel<<<mv_grid(n_tasks, max_n, 4), MV_THREADS, 0, (cudaStream_t)stream>>>(task_dev, SRC, DST);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_take_blocks_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                                    const int64_t *idx_dev, const double *SRC, double *DST, b200_stream_t stream) {
    if (n_tasks <= 0) return B200_OK;
    if (n_tasks > 65535) return set_error(B200_ERR_ARG, "too many take tasks (%lld)", (long long)n_tasks);
    int64_t max_n = 0;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t *rec = task_host + t * B200_TAKE_REC;
        int64_t n = rec[2] * rec[3] * rec[4];
        if (n > max_n) max_n = n;
    }
    if (max_n == 0) return B200_OK;
    take_blocks_kernel<<<mv_grid(n_tasks, max_n, 4), MV_THREADS, 0, (cudaStream_t)stream>>>(task_dev, idx_dev, SRC, DST);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_scale_axis_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                                   const double *S_dev, double *X, b200_stream_t stream) {
    if (n_tasks <= 0) return B200_OK;
    if (n_tasks > 65535) return set_error(B200_ERR_ARG, "too many scale tasks (%lld)", (long long)n_tasks);
    int64_t max_n = 0;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t *rec = task_host + t * B200_SCALE_REC;
        int64_t n = rec[1] * rec[2] * rec[3];
        if (n > max_n) max_n = n;
    }
    if (max_n == 0) return B200_OK;
    scale_axis_kernel<<<mv_grid(n_tasks, max_n, 4), MV_THREADS, 0, (cudaStream_t)stream>>>(task_dev, S_dev, X);
    B200_CHECK_LAUNCH();
    return B200_OK;
}
