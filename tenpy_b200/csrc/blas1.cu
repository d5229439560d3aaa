// blas1.cu -- Lanczos vector operations on packed block buffers (HBM-bandwidth bound).
//
// Replaces the per-block BLAS-1 loops of the reference: Array_iadd_prefactor_other (pyx:860, daxpy
// pyx:328), Array_iscale_prefactor (pyx:964, dscal pyx:350), _inner_worker (pyx:1791, ddot pyx:1854) and
// Array.norm (npc:2241).  Because an Array lives in ONE packed buffer whose padding is zero, an op between
// two Arrays with the same block table is a single pass over the whole buffer; Arrays with different block
// tables use the *_segments variants driven by a device-resident (x_off, y_off, len) table.
#include "common.cuh"

namespace b200 {

constexpr int B1_THREADS = 256;

static inline int b1_grid(int64_t n, int per_thread) {
    int64_t blocks = (n + (int64_t)B1_THREADS * per_thread - 1) / ((int64_t)B1_THREADS * per_thread);
    int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

__global__ void __launch_bounds__(B1_THREADS) axpy_kernel(int64_t n, double alpha, const double *__restrict__ x,
                                                          double *__restrict__ y) {
    const int64_t n2 = n >> 1;
    const bool al = ((((uintptr_t)x) | ((uintptr_t)y)) & 15) == 0;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (al) {
        const double2 *x2 = reinterpret_cast<const double2 *>(x);
        double2 *y2 = reinterpret_cast<double2 *>(y);
        for (int64_t j = i; j < n2; j += stride) {
            double2 a = x2[j], b = y2[j];
            b.x = fma(alpha, a.x, b.x);
            b.y = fma(alpha, a.y, b.y);
            y2[j] = b;
        }
        if (i == 0 && (n & 1)) y[n - 1] = fma(alpha, x[n - 1], y[n - 1]);
    } else {
        for (int64_t j = i; j < n; j += stride) y[j] = fma(alpha, x[j], y[j]);
    }
}

__global__ void __launch_bounds__(B1_THREADS) scal_kernel(int64_t n, double alpha, double *__restrict__ x) {
    const int64_t n2 = n >> 1;
    const bool al = (((uintptr_t)x) & 15) == 0;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (al) {
        double2 *x2 = reinterpret_cast<double2 *>(x);
        for (int64_t j = i; j < n2; j += stride) {
            double2 a = x2[j];
            a.x *= alpha;
            a.y *= alpha;
            x2[j] = a;
        }
        if (i == 0 && (n & 1)) x[n - 1] *= alpha;
    } else {
        for (int64_t j = i; j < n; j += stride) x[j] *= alpha;
    }
}

// stage 1 of the deterministic dot: one partial per CTA
__global__ void __launch_bounds__(B1_THREADS) dot_partial_kernel(int64_t n, const double *__restrict__ x,
                                                                 const double *__restrict__ y,
                                                                 double *__restrict__ partial) {
    __shared__ double red[32];
    const int64_t n2 = n >> 1;
    const bool al = ((((uintptr_t)x) | ((uintptr_t)y)) & 15) == 0;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    double s0 = 0.0, s1 = 0.0;
    if (al) {
        const double2 *x2 = reinterpret_cast<const double2 *>(x);
        const double2 *y2 = reinterpret_cast<const double2 *>(y);
        for (int64_t j = i; j < n2; j += stride) {
            double2 a = x2[j], b = y2[j];
            s0 = fma(a.x, b.x, s0);
            s1 = fma(a.y, b.y, s1);
        }
        if (i == 0 && (n & 1)) s0 = fma(x[n - 1], y[n - 1], s0);
    } else {
        for (int64_t j = i; j < n; j += stride) s0 = fma(x[j], y[j], s0);
    }
    double s = block_sum(s0 + s1, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// stage 2: fixed-order sum of the partials by one CTA
__global__ void __launch_bounds__(B1_THREADS) dot_final_kernel(int np, const double *__restrict__ partial,
                                                               double *__restrict__ out) {
    __shared__ double red[32];
    double s = 0.0;
    for (int j = threadIdx.x; j < np; j += blockDim.x) s += partial[j];
    s = block_sum(s, red);
    if (threadIdx.x == 0) out[0] = s;
}

// w -= alpha*v1 + beta*v0 ; partial |w|^2
__global__ void __launch_bounds__(B1_THREADS) lanczos_update_kernel(int64_t n, double alpha,
                                                                    const double *__restrict__ v1, double beta,
                                                                    const double *__restrict__ v0,
                                                                    double *__restrict__ w,
                                                                    double *__restrict__ partial) {
    __shared__ double red[32];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    double s = 0.0;
    for (int64_t j = i; j < n; j += stride) {
        double r = w[j];
        r = fma(-alpha, v1[j], r);
        if (v0) r = fma(-beta, v0[j], r);
        w[j] = r;
        s = fma(r, r, s);
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// the same step with the scalars left on the device: alpha = *alpha_p, beta = sqrt(*beta2_p) (beta2_p / v0 may be null).
// sqrt and the division below are IEEE correctly rounded for double: bit-identical to the host-scalar route.
__global__ void __launch_bounds__(B1_THREADS) lanczos_update_dev_kernel(int64_t n, const double *__restrict__ alpha_p,
                                                                        const double *__restrict__ v1,
                                                                        const double *__restrict__ beta2_p,
                                                                        const double *__restrict__ v0,
                                                                        double *__restrict__ w,
                                                                        double *__restrict__ partial) {
    __shared__ double red[32];
    const double alpha = alpha_p[0];
    const bool have0 = (v0 != nullptr) && (beta2_p != nullptr);
    const double beta = have0 ? sqrt(beta2_p[0]) : 0.0;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    double s = 0.0;
    for (int64_t j = i; j < n; j += stride) {
        double r = w[j];
        r = fma(-alpha, v1[j], r);
        if (have0) r = fma(-beta, v0[j], r);
        w[j] = r;
        s = fma(r, r, s);
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// x *= 1 / sqrt(*norm2_p)
__global__ void __launch_bounds__(B1_THREADS) scal_rsqrt_dev_kernel(int64_t n, const double *__restrict__ norm2_p,
                                                                    double *__restrict__ x) {
    const double a = 1.0 / sqrt(norm2_p[0]);
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
        x[j] *= a;
}

// segment kernels: blockIdx.y = segment, blockIdx.x strides over the segment
__global__ void __launch_bounds__(B1_THREADS) axpy_seg_kernel(const int64_t *__restrict__ seg, double alpha,
                                                              const double *__restrict__ x, double *__restrict__ y) {
    const int64_t xo = seg[3 * blockIdx.y], yo = seg[3 * blockIdx.y + 1], len = seg[3 * blockIdx.y + 2];
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < len; j += (int64_t)gridDim.x * blockDim.x)
        y[yo + j] = fma(alpha, x[xo + j], y[yo + j]);
}

__global__ void __launch_bounds__(B1_THREADS) dot_seg_kernel(const int64_t *__restrict__ seg,
                                                             const double *__restrict__ x,
                                                             const double *__restrict__ y,
                                                             double *__restrict__ partial) {
    __shared__ double red[32];
    const int64_t xo = seg[3 * blockIdx.y], yo = seg[3 * blockIdx.y + 1], len = seg[3 * blockIdx.y + 2];
    double s = 0.0;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < len; j += (int64_t)gridDim.x * blockDim.x)
        s = fma(x[xo + j], y[yo + j], s);
    s = block_sum(s, red);
    if (threadIdx.x == 0) partial[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
}

// out = sum_k c_k v_k for complex c_k (coef[2k] + i coef[2k+1]); v_k one plane (real, in_planes = 1) or the planes
// [re; im] of a packed complex vector (in_planes = 2); out is always [re; im].  One thread per element, the sum over k in
// the order of the table, so that a result does not depend on the launch geometry.
constexpr int KC_MAX_VEC = 64;

__global__ void __launch_bounds__(B1_THREADS) krylov_combine_kernel(int64_t n, int nvec, int in_planes,
                                                                    const double *const *__restrict__ v,
                                                                    const double *__restrict__ coef,
                                                                    double *__restrict__ out) {
    __shared__ double c[2 * KC_MAX_VEC];
    __shared__ const double *vp[KC_MAX_VEC];
    for (int t = threadIdx.x; t < 2 * nvec; t += blockDim.x) c[t] = coef[t];
    for (int t = threadIdx.x; t < nvec; t += blockDim.x) vp[t] = v[t];
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    double re = 0.0, im = 0.0;
    if (in_planes == 2) {
        for (int k = 0; k < nvec; ++k) {
            const double xr = vp[k][j], xi = vp[k][n + j], cr = c[2 * k], ci = c[2 * k + 1];
            re = fma(cr, xr, re);
            re = fma(-ci, xi, re);
            im = fma(cr, xi, im);
            im = fma(ci, xr, im);
        }
    } else {
        for (int k = 0; k < nvec; ++k) {
            const double x = vp[k][j];
            re = fma(c[2 * k], x, re);
            im = fma(c[2 * k + 1], x, im);
        }
    }
    out[j] = re;
    out[n + j] = im;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_axpy_f64(int64_t n, double alpha, const double *X, double *Y, b200_stream_t stream) {
    if (n <= 0) return B200_OK;
    axpy_kernel<<<b1_grid(n, 8), B1_THREADS, 0, (cudaStream_t)stream>>>(n, alpha, X, Y);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_scal_f64(int64_t n, double alpha, double *X, b200_stream_t stream) {
    if (n <= 0) return B200_OK;
    scal_kernel<<<b1_grid(n, 8), B1_THREADS, 0, (cudaStream_t)stream>>>(n, alpha, X);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_dot_f64(int64_t n, const double *X, const double *Y, double *scratch, double *out,
                            b200_stream_t stream) {
    int grid = b1_grid(n, 8);
    if (grid > B200_DOT_SCRATCH) grid = B200_DOT_SCRATCH;
    if (n <= 0) {
        B200_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), (cudaStream_t)stream));
        return B200_OK;
    }
    dot_partial_kernel<<<grid, B1_THREADS, 0, (cudaStream_t)stream>>>(n, X, Y, scratch);
    B200_CHECK_LAUNCH();
    dot_final_kernel<<<1, B1_THREADS, 0, (cudaStream_t)stream>>>(grid, scratch, out);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_lanczos_update_f64(int64_t n, double alpha, const double *V1, double beta, const double *V0,
                                       double *W, double *scratch, double *out, b200_stream_t stream) {
    int grid = b1_grid(n, 8);
    if (grid > B200_DOT_SCRATCH) grid = B200_DOT_SCRATCH;
    if (n <= 0) {
        B200_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), (cudaStream_t)stream));
        return B200_OK;
    }
    lanczos_update_kernel<<<grid, B1_THREADS, 0, (cudaStream_t)stream>>>(n, alpha, V1, beta, V0, W, scratch);
    B200_CHECK_LAUNCH();
    dot_final_kernel<<<1, B1_THREADS, 0, (cudaStream_t)stream>>>(grid, scratch, out);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_lanczos_update_dev_f64(int64_t n, const double *alpha_dev, const double *V1, const double *beta2_dev,
                                           const double *V0, double *W, double *scratch, double *out,
                                           b200_stream_t stream) {
    int grid = b1_grid(n, 8);
    if (grid > B200_DOT_SCRATCH) grid = B200_DOT_SCRATCH;
    if (n <= 0) {
        B200_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), (cudaStream_t)stream));
        return B200_OK;
    }
    lanczos_update_dev_kernel<<<grid, B1_THREADS, 0, (cudaStream_t)stream>>>(n, alpha_dev, V1, beta2_dev, V0, W, scratch);
    B200_CHECK_LAUNCH();
    dot_final_kernel<<<1, B1_THREADS, 0, (cudaStream_t)stream>>>(grid, scratch, out);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_scal_rsqrt_dev_f64(int64_t n, const double *norm2_dev, double *X, b200_stream_t stream) {
    if (n <= 0) return B200_OK;
    scal_rsqrt_dev_kernel<<<b1_grid(n, 8), B1_THREADS, 0, (cudaStream_t)stream>>>(n, norm2_dev, X);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

static inline int seg_grid_x(int64_t n_seg, int64_t max_len) {
    int64_t gx = (max_len + (int64_t)B1_THREADS * 4 - 1) / ((int64_t)B1_THREADS * 4);
    if (gx < 1) gx = 1;
    int64_t cap = B200_DOT_SCRATCH / (n_seg > 0 ? n_seg : 1);
    if (cap < 1) cap = 1;
    if (gx > cap) gx = cap;
    return (int)gx;
}

extern "C" int b200_axpy_segments_f64(int64_t n_seg, const int64_t *seg_dev, int64_t max_len, double alpha,
                                      const double *X, double *Y, b200_stream_t stream) {
    if (n_seg <= 0 || max_len <= 0) return B200_OK;
    if (n_seg > 65535) return set_error(B200_ERR_ARG, "too many segments (%lld)", (long long)n_seg);
    int64_t gx = (max_len + (int64_t)B1_THREADS * 4 - 1) / ((int64_t)B1_THREADS * 4);
    if (gx > 1024) gx = 1024;
    dim3 grid((unsigned)gx, (unsigned)n_seg);
    axpy_seg_kernel<<<grid, B1_THREADS, 0, (cudaStream_t)stream>>>(seg_dev, alpha, X, Y);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_dot_segments_f64(int64_t n_seg, const int64_t *seg_dev, int64_t max_len, const double *X,
                                     const double *Y, double *scratch, double *out, b200_stream_t stream) {
    if (n_seg <= 0 || max_len <= 0) {
        B200_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), (cudaStream_t)stream));
        return B200_OK;
    }
    if (n_seg > B200_DOT_SCRATCH) return set_error(B200_ERR_ARG, "too many segments (%lld)", (long long)n_seg);
    int gx = seg_grid_x(n_seg, max_len);
    dim3 grid((unsigned)gx, (unsigned)n_seg);
    dot_seg_kernel<<<grid, B1_THREADS, 0, (cudaStream_t)stream>>>(seg_dev, X, Y, scratch);
    B200_CHECK_LAUNCH();
    dot_final_kernel<<<1, B1_THREADS, 0, (cudaStream_t)stream>>>((int)(gx * n_seg), scratch, out);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_krylov_combine_f64(int64_t n, int64_t nvec, int64_t in_planes, const double *const *V_dev,
                                       const double *const *V_host, const double *coef_dev, double *OUT,
                                       b200_stream_t stream) {
    if (nvec < 1 || nvec > KC_MAX_VEC) return set_error(B200_ERR_ARG, "krylov_combine: nvec = %lld outside 1..%d",
                                                        (long long)nvec, KC_MAX_VEC);
    if (in_planes != 1 && in_planes != 2)
        return set_error(B200_ERR_ARG, "krylov_combine: in_planes = %lld (1 or 2)", (long long)in_planes);
    if (n < 0) return set_error(B200_ERR_ARG, "krylov_combine: n = %lld < 0", (long long)n);
    if (n == 0) return B200_OK;
    if (!V_dev || !V_host || !coef_dev || !OUT) return set_error(B200_ERR_ARG, "krylov_combine: null pointer");
    const uintptr_t o0 = (uintptr_t)OUT, o1 = o0 + (uintptr_t)(2 * n) * sizeof(double);
    for (int64_t k = 0; k < nvec; ++k) {
        const uintptr_t v0 = (uintptr_t)V_host[k], v1 = v0 + (uintptr_t)(in_planes * n) * sizeof(double);
        if (!V_host[k]) return set_error(B200_ERR_ARG, "krylov_combine: vector %lld is null", (long long)k);
        if (v0 < o1 && o0 < v1) return set_error(B200_ERR_ARG, "krylov_combine: out overlaps vector %lld", (long long)k);
    }
    const int64_t blocks = (n + B1_THREADS - 1) / B1_THREADS;
    if (blocks > 0x7fffffffLL) return set_error(B200_ERR_ARG, "krylov_combine: n = %lld too large", (long long)n);
    krylov_combine_kernel<<<(unsigned)blocks, B1_THREADS, 0, (cudaStream_t)stream>>>(n, (int)nvec, (int)in_planes,
                                                                                     V_dev, coef_dev, OUT);
    B200_CHECK_LAUNCH();
    return B200_OK;
}
