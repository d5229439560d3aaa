// ozaki.cu -- FP64 matrix products on the int8 tensor path of the H100 (wgmma.mma_async s8 x s8, int32 accumulation in
// registers), for the chi^3 contractions of the effective-H matvec and the environment updates.
//
// Replaces (for large dense blocks) the level-wise dgemm of CblasGemmBatch.run, tenpy/linalg/_npc_helper.pyx:204-274,
// reached from _tensordot_worker pyx:1498-1790 / np_conserved.py:4846.
//
// Scheme (Ozaki splitting, error-free int8 slices):
//   every row i of A (and every column j of B) is scaled by a power of two 2^-ea_i (2^-eb_j) so that |x| < 1, and
//   written as   x = sum_t d_t 2^(-6-7t) + r,   d_t in [-64, 64] (signed 7-bit digits, round to nearest), t < s,
//   |r| <= 2^(-7 s).  Then
//       (A B)_ij = 2^(ea_i + eb_j - 12) sum_{d=0}^{s-1} 2^(-7 d) C_d,      C_d = sum_{t+u=d} A_t B_u   (int8 x int8 -> int32)
//   up to the dropped slice products t + u >= s.  Every C_d is an EXACT integer matrix (k * 2^12 * (d+1) < 2^31), computed
//   by wgmma on 128 x 64 tiles with the accumulators in registers; the diagonals are summed in FP64 in the epilogue.
//   s = 7 gives ~1e-14 relative to (|A||B|)_ij, s = 8 FP64 rounding level (tests/test_ozaki.py).
//
// Data layout.  A split operand ("panel layout") is, per slice t and per tile of 128 rows, the sequence of its 16-byte
// k-chunks, each chunk stored as 128 rows x 16 bytes (2 KB):   [slice][row tile][k chunk][row in tile][16 B].
// A stage of the pipeline (4 consecutive k-chunks of one row tile of one slice = 8 KB, contiguous in HBM) is brought in
// by bulk async copies of the TMA unit (cp.async.bulk) and is directly the un-swizzled K-major core-matrix layout wgmma
// reads: core matrix (8 rows x 16 B) contiguous, LBO (K direction) = chunk stride, SBO (row direction) = 128 B.
//
// Kernel (persistent, one CTA per SM, 3 warpgroups): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = MMA
// and epilogue, each owning 64 rows x 64 columns of the 128 x 64 output tile (the B operand is read as one half of its
// 128-row panel tile).  A thread holds 4 int32 accumulators of 32 registers, so the diagonals are processed in passes of
// up to 4, least significant pass first and the groups aligned at the top (s = 7: d = 3..6 then d = 0..2): the last pass
// needs the fewest slices; within a pass every loaded slice tile is reused by up to 4 MMAs.  The FP64 summation of a pass
// is the same sequence of operations for every element whatever the tile shape, so results do not depend on it.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "tc05.cuh"

namespace b200 {

namespace {

constexpr int OZ_MAX_SLICES = 10;
constexpr int OZ_TILE = 128;               // rows per tile (M and N)
constexpr int OZ_CHUNK_BYTES = 16 * OZ_TILE;  // one k-chunk of one row tile: 128 rows x 16 B
constexpr int OZ_SMEM_BUDGET = 224 * 1024;

__host__ __device__ inline int64_t oz_row_tiles(int64_t rows) { return (rows + OZ_TILE - 1) / OZ_TILE; }
__host__ __device__ inline int64_t oz_k_chunks(int64_t k) { return (k + 63) / 64 * 4; }   // K padded to 64 bytes

// byte offsets inside a split buffer: digits | scales (double per padded row) | max bits (u64 per padded row)
struct SplitLayout {
    int64_t rt, kc, digits_bytes, scale_off, max_off, total;
};
__host__ inline SplitLayout split_layout(int64_t rows, int64_t k, int slices) {
    SplitLayout L;
    L.rt = oz_row_tiles(rows);
    L.kc = oz_k_chunks(k);
    L.digits_bytes = (int64_t)slices * L.rt * L.kc * OZ_CHUNK_BYTES;
    L.scale_off = (L.digits_bytes + 255) / 256 * 256;
    L.max_off = L.scale_off + L.rt * OZ_TILE * 8;
    L.total = L.max_off + L.rt * OZ_TILE * 8;
    return L;
}

// ---- pass 1 of the split: max |x| per row (as the bit pattern of a non-negative double: integer order = value order) ---
// rows contiguous in k (ld_k == 1): one warp per row
__global__ void oz_rowmax_kcontig_kernel(const double *__restrict__ X, int64_t rows, int64_t k, int64_t ld_row,
                                         unsigned long long *__restrict__ maxbits) {
    int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= rows) return;
    const double *x = X + r * ld_row;
    double m = 0.0;
    for (int64_t i = threadIdx.x & 31; i < k; i += 32) m = fmax(m, fabs(x[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) maxbits[r] = (unsigned long long)__double_as_longlong(m);
}
// rows strided in k (ld_row == 1): 32 rows x 8 k-lanes per block, grid.y splits k; combined with atomicMax
__global__ void oz_rowmax_rcontig_kernel(const double *__restrict__ X, int64_t rows, int64_t k, int64_t ld_k,
                                         int64_t k_per_block, unsigned long long *__restrict__ maxbits) {
    __shared__ double red[8][33];
    int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    int64_t r = (int64_t)blockIdx.x * 32 + tx;
    int64_t k0 = (int64_t)blockIdx.y * k_per_block, k1 = min(k, k0 + k_per_block);
    double m = 0.0;
    if (r < rows)
        for (int64_t i = k0 + ty; i < k1; i += 8) m = fmax(m, fabs(X[i * ld_k + r]));
    red[ty][tx] = m;
    __syncthreads();
    if (ty == 0 && r < rows) {
#pragma unroll
        for (int j = 1; j < 8; ++j) m = fmax(m, red[j][tx]);
        atomicMax(maxbits + r, (unsigned long long)__double_as_longlong(m));
    }
}

// ---- pass 2 of the split: digits.  One thread = one row x one 16-byte k-chunk (16 elements), all slices. ---------------
// scale[r] = 2^e with |x| 2^-e < 1 for the whole row (e = exponent of the row maximum + 1); zero rows: scale 1.
__global__ void oz_split_kernel(const double *__restrict__ X, int64_t rows, int64_t k, int64_t ld_row, int64_t ld_k,
                                int slices, int64_t rt_count, int64_t kc_count,
                                const unsigned long long *__restrict__ maxbits, double *__restrict__ scale,
                                uint8_t *__restrict__ digits) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;       // padded row index
    int64_t c = blockIdx.y;                                           // k chunk
    if (r >= rt_count * OZ_TILE) return;
    uint32_t packed[OZ_MAX_SLICES][4];
#pragma unroll
    for (int t = 0; t < OZ_MAX_SLICES; ++t) packed[t][0] = packed[t][1] = packed[t][2] = packed[t][3] = 0u;
    if (r < rows) {
        unsigned long long mb = maxbits[r];
        int be = (int)((mb >> 52) & 0x7ff);                          // biased exponent of the row maximum
        be = min(max(be, 64), 1980);                                 // keep 2^e, 2^-e and their products finite normals
        double sc = 1.0, inv64 = 64.0;
        if (mb != 0ull) {
            // scale = 2^(be - 1023 + 1); inv = 2^-(be - 1022); digits of x * inv * 64
            sc = __longlong_as_double((long long)(be + 1) << 52);
            inv64 = __longlong_as_double((long long)(2046 - (be + 1) + 6) << 52);
        }
        if (c == 0) scale[r] = sc;
        const double *x = X + r * ld_row + c * 16 * ld_k;
        int64_t kleft = k - c * 16;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            double v = (i < kleft) ? x[i * ld_k] * inv64 : 0.0;
#pragma unroll
            for (int t = 0; t < OZ_MAX_SLICES; ++t) {
                if (t < slices) {
                    double d = rint(v);
                    v = (v - d) * 128.0;
                    packed[t][i >> 2] |= ((uint32_t)(int)d & 0xffu) << (8 * (i & 3));
                }
            }
        }
    } else if (c == 0) {
        scale[r] = 1.0;
    }
    int64_t rt = r / OZ_TILE, rr = r % OZ_TILE;
#pragma unroll
    for (int t = 0; t < OZ_MAX_SLICES; ++t) {
        if (t < slices) {
            uint8_t *dst = digits + (((int64_t)t * rt_count + rt) * kc_count + c) * OZ_CHUNK_BYTES + rr * 16;
            *reinterpret_cast<uint4 *>(dst) = make_uint4(packed[t][0], packed[t][1], packed[t][2], packed[t][3]);
        }
    }
}

// ---- single-launch split (slices <= OZ_FUSED_MAX_SLICES): row maximum and digits in one kernel ---------------------------
// One CTA = 32 rows x all k.  Phase 1 streams the rows once for the maximum; phase 2 re-reads them (from L2: the CTA has
// just touched these 32 k doubles) in blocks of 128 k through shared memory, so that both the global reads and the 16-byte
// digit stores are coalesced for either operand orientation.  The digits come from ONE conversion per element:
//   X = rint(x 2^-e 2^(6 + 7 (s-1)))  (int64, |X| <= 2^(6 + 7 (s-1)) <= 2^62),   X = sum_t d_t 128^(s-1-t),
// peeled off from the least significant end with d_t in [-64, 63] (t > 0) and the carry into the next digit; the top digit
// is in [-64, 64].  This is the same number as the round-to-nearest expansion of oz_split_kernel (a different, equally exact
// signed-digit string when a remainder is exactly one half).
constexpr int OZ_FUSED_MAX_SLICES = 9;
constexpr int OZF_ROWS = 16, OZF_KB = 256, OZF_THREADS = 256;      // 16 rows x 16 chunks of 16 k per block of the k loop

template <bool KCONTIG>
__global__ void __launch_bounds__(OZF_THREADS, 2) oz_split_fused_kernel(const double *__restrict__ X, int64_t rows, int64_t k,
                                                                        int64_t ld, int slices, int64_t rt_count, int64_t kc_count,
                                                                        double *__restrict__ scale, uint8_t *__restrict__ digits) {
    // KCONTIG: element (r, kk) = X[r * ld + kk], tile in shared memory [row][OZF_KB + 1]
    // else:    element (r, kk) = X[kk * ld + r], tile in shared memory [kk][OZF_ROWS]
    __shared__ double sx[OZF_ROWS * (OZF_KB + 1)];
    __shared__ double red[OZF_THREADS / OZF_ROWS][OZF_ROWS];
    __shared__ double s_mul[OZF_ROWS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rr = tid % OZF_ROWS, cc = tid / OZF_ROWS;               // row of the CTA / k lane (0..15)
    const int64_t r0 = (int64_t)blockIdx.x * OZF_ROWS;
    // ---- phase 1: max |x| of every row (independent loads, 8 in flight per thread)
    if (KCONTIG) {
#pragma unroll
        for (int j = 0; j < OZF_ROWS / 8; ++j) {
            const int lr = warp + 8 * j;
            double m = 0.0;
            if (r0 + lr < rows) {
                const double *x = X + (r0 + lr) * ld;
                int64_t i = lane;
                for (; i + 7 * 32 < k; i += 8 * 32) {
                    double v[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) v[u] = x[i + 32 * u];
#pragma unroll
                    for (int u = 0; u < 8; ++u) m = fmax(m, fabs(v[u]));
                }
                for (; i < k; i += 32) m = fmax(m, fabs(x[i]));
            }
            m = warp_max(m);
            if (lane == 0) red[0][lr] = m;
        }
        __syncthreads();
    } else {
        double m = 0.0;
        if (r0 + rr < rows) {
            const double *x = X + r0 + rr;
            int64_t kk = cc;
            for (; kk + 7 * 16 < k; kk += 8 * 16) {
                double v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = x[(kk + 16 * u) * ld];
#pragma unroll
                for (int u = 0; u < 8; ++u) m = fmax(m, fabs(v[u]));
            }
            for (; kk < k; kk += 16) m = fmax(m, fabs(x[kk * ld]));
        }
        red[cc][rr] = m;
        __syncthreads();
        if (tid < OZF_ROWS) {
#pragma unroll
            for (int j = 1; j < OZF_THREADS / OZF_ROWS; ++j) m = fmax(m, red[j][tid]);
            red[0][tid] = m;
        }
        __syncthreads();
    }
    if (tid < OZF_ROWS) {
        const unsigned long long mb = (unsigned long long)__double_as_longlong(red[0][tid]);
        int be = (int)((mb >> 52) & 0x7ff);                          // biased exponent of the row maximum
        be = min(max(be, 64), 1980);                                 // keep 2^e, 2^-e and their products finite normals
        double sc = 1.0, mul = 0.0;
        if (mb != 0ull) {
            sc = __longlong_as_double((long long)(be + 1) << 52);    // 2^e, e = be - 1022: |x| 2^-e < 1
            mul = __longlong_as_double((long long)(2051 - be + 7 * (slices - 1)) << 52);   // 2^(-e + 6 + 7 (s-1))
        }
        s_mul[tid] = mul;
        scale[r0 + tid] = sc;                                        // the grid covers exactly the padded rows
    }
    __syncthreads();
    // ---- phase 2: digits, 256 k at a time
    const double mul = s_mul[rr];
    const int64_t r = r0 + rr;
    const int64_t rt = r / OZ_TILE, rin = r % OZ_TILE;
    const int64_t kpad = kc_count * 16;
    for (int64_t kb = 0; kb < kpad; kb += OZF_KB) {
        if (KCONTIG) {
#pragma unroll
            for (int j = 0; j < OZF_ROWS / 8; ++j) {
                const int lr = warp + 8 * j;
                const bool rok = r0 + lr < rows;
                const double *x = X + (r0 + lr) * ld + kb;
#pragma unroll
                for (int i = 0; i < OZF_KB / 32; ++i) {
                    const int kk = lane + 32 * i;
                    sx[lr * (OZF_KB + 1) + kk] = (rok && kb + kk < k) ? x[kk] : 0.0;
                }
            }
        } else {
            const bool rok = r0 + rr < rows;
#pragma unroll
            for (int j = 0; j < OZF_KB / 16; ++j) {
                const int kk = cc + 16 * j;
                sx[kk * OZF_ROWS + rr] = (rok && kb + kk < k) ? X[(kb + kk) * ld + r0 + rr] : 0.0;
            }
        }
        __syncthreads();
        const int64_t c = kb / 16 + cc;
        if (c < kc_count) {
            uint32_t packed[OZ_FUSED_MAX_SLICES][4];
#pragma unroll
            for (int t = 0; t < OZ_FUSED_MAX_SLICES; ++t) packed[t][0] = packed[t][1] = packed[t][2] = packed[t][3] = 0u;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const double v = (KCONTIG ? sx[rr * (OZF_KB + 1) + cc * 16 + i] : sx[(cc * 16 + i) * OZF_ROWS + rr]) * mul;
                long long xi = __double2ll_rn(v);
#pragma unroll
                for (int t = OZ_FUSED_MAX_SLICES - 1; t >= 1; --t) {
                    if (t < slices) {
                        const int d = (int)((xi + 64) & 127) - 64;
                        xi = (xi - d) >> 7;
                        packed[t][i >> 2] |= ((uint32_t)d & 0xffu) << (8 * (i & 3));
                    }
                }
                packed[0][i >> 2] |= ((uint32_t)(int)xi & 0xffu) << (8 * (i & 3));
            }
#pragma unroll
            for (int t = 0; t < OZ_FUSED_MAX_SLICES; ++t) {
                if (t < slices) {
                    uint8_t *dst = digits + (((int64_t)t * rt_count + rt) * kc_count + c) * OZ_CHUNK_BYTES + rin * 16;
                    *reinterpret_cast<uint4 *>(dst) = make_uint4(packed[t][0], packed[t][1], packed[t][2], packed[t][3]);
                }
            }
        }
        __syncthreads();
    }
}

// ---- the tensor-core kernel ---------------------------------------------------------------------------------------------
struct OzGemmArgs {
    const uint8_t *As, *Bs;      // digits of the split operands
    const double *sA, *sB;       // row scales 2^ea_i, 2^eb_j
    double *C;
    int64_t ldc;
    int32_t M, N;                // valid extents of C
    int32_t kc;                  // k chunks (16 B) of both operands, multiple of 4
    int32_t rta, rtb;            // row tiles of A / B
    int32_t slices;
    int32_t cps;                 // k chunks per pipeline stage (4 or 2)
    int32_t nstages;
    int32_t accumulate;          // 0: C = A.B, 1: C += A.B
    int32_t *abort_flag;
    long long *dbg;              // optional (B200_OZ_DEBUG): cycle counters of CTA 0, see b200_ozaki_mm_f64
};

constexpr int OZ_TN = 64;                   // columns of C per CTA tile: one half of a 128-row tile of B
constexpr int OZ_THREADS = 384;             // warpgroup 0: producer (one thread), warpgroups 1-2: MMA + epilogue
constexpr int OZ_CONSUMER_THREADS = 256;    // each consumer warpgroup owns 64 rows x 64 columns of the tile
constexpr int OZ_MAX_STAGES = 4;

__device__ __forceinline__ double oz_i2d(uint32_t r) { return (double)(int32_t)r; }

__global__ void __launch_bounds__(OZ_THREADS, 1) oz_gemm_kernel(OzGemmArgs p) {
    extern __shared__ __align__(1024) uint8_t oz_smem[];
    __shared__ uint64_t full_bar[OZ_MAX_STAGES], empty_bar[OZ_MAX_STAGES];
    using namespace sm90;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = p.slices, cps = p.cps, nst = p.nstages;
    const uint32_t a_bytes = (uint32_t)cps * OZ_CHUNK_BYTES;          // A slice tile of a stage: cps chunks x 128 rows
    const uint32_t b_bytes = a_bytes / 2;                             // B slice half tile: cps chunks x 64 rows
    const uint32_t stage_bytes = (uint32_t)s * (a_bytes + b_bytes);
    const int npass = (s + 3) / 4;
    const int ksteps = p.kc / cps;                                    // pipeline stages per pass
    const int mt_count = (p.M + OZ_TILE - 1) / OZ_TILE, nt_count = (p.N + OZ_TN - 1) / OZ_TN;
    const int ntiles = mt_count * nt_count;

    if (threadIdx.x == 0) {
        for (int i = 0; i < nst; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], OZ_CONSUMER_THREADS);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 0) {
        if (lane != 0) return;
        // ================= producer: bulk copies of slice tiles =================
        uint32_t it = 0;
        bool ok = true;
        long long t_wait = 0, t0 = clock64();
        for (int tile = blockIdx.x; tile < ntiles && ok; tile += gridDim.x) {
            const int mt = tile % mt_count, nt = tile / mt_count;
            const int bt = nt >> 1, bhalf = nt & 1;
            for (int g = npass - 1; g >= 0 && ok; --g) {
                const int nsl = s - 4 * (npass - 1 - g);             // slices 0 .. nsl-1 of both operands are needed (= d_hi + 1)
                for (int ks = 0; ks < ksteps; ++ks, ++it) {
                    const int slot = it % nst;
                    const long long tw = clock64();
                    ok = mbar_wait(&empty_bar[slot], ((it / nst) & 1) ^ 1, p.abort_flag);
                    t_wait += clock64() - tw;
                    if (!ok) break;
                    mbar_expect_tx(&full_bar[slot], (uint32_t)nsl * (a_bytes + b_bytes));
                    uint8_t *st = oz_smem + (size_t)slot * stage_bytes;
                    for (int t = 0; t < nsl; ++t) {
                        const uint8_t *ga = p.As + (((int64_t)t * p.rta + mt) * p.kc + (int64_t)ks * cps) * OZ_CHUNK_BYTES;
                        const uint8_t *gb = p.Bs + (((int64_t)t * p.rtb + bt) * p.kc + (int64_t)ks * cps) * OZ_CHUNK_BYTES +
                                            bhalf * (OZ_CHUNK_BYTES / 2);
                        bulk_g2s(st + (size_t)t * a_bytes, ga, a_bytes, &full_bar[slot]);
                        uint8_t *sb = st + (size_t)s * a_bytes + (size_t)t * b_bytes;
                        for (int c = 0; c < cps; ++c)
                            bulk_g2s(sb + c * (OZ_CHUNK_BYTES / 2), gb + (size_t)c * OZ_CHUNK_BYTES, OZ_CHUNK_BYTES / 2,
                                     &full_bar[slot]);
                    }
                }
            }
        }
        if (p.dbg && blockIdx.x == 0) {
            p.dbg[0] = clock64() - t0;
            p.dbg[1] = t_wait;
        }
        return;
    }
    if (warp < 4) return;

    // ================= consumers: wgmma into register accumulators, epilogue straight from the registers =================
    const int cw = (warp >> 2) - 1;                                   // rows [64 cw, 64 cw + 64) of the 128-row tile
    const int wl = warp & 3;
    uint32_t acc[4][32];                                              // one int32 accumulator per diagonal of a pass
    uint32_t it = 0;
    bool ok = true;
    long long t_full = 0, t_epi = 0, t0 = clock64();
    for (int tile = blockIdx.x; tile < ntiles && ok; tile += gridDim.x) {
        const int mt = tile % mt_count, nt = tile / mt_count;
        for (int g = npass - 1; g >= 0 && ok; --g) {
            const int d_hi = s - 1 - 4 * (npass - 1 - g), d_lo = max(0, d_hi - 3);
            for (int ks = 0; ks < ksteps; ++ks, ++it) {
                const int slot = it % nst;
                const long long tw = clock64();
                ok = mbar_wait(&full_bar[slot], (it / nst) & 1, p.abort_flag);
                t_full += clock64() - tw;
                if (!ok) break;
                const uint32_t sa = smem_addr(oz_smem + (size_t)slot * stage_bytes) + (uint32_t)cw * 64u * 16u;
                const uint32_t sb = smem_addr(oz_smem + (size_t)slot * stage_bytes + (size_t)s * a_bytes);
                wgmma_fence();
                for (int kk = 0; kk < cps / 2; ++kk) {                // one wgmma covers 32 bytes of K = two chunks
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int d = d_lo + j;
                        if (d > d_hi) break;
                        for (int t = 0; t <= d; ++t) {                // all pairs (t, u = d - t) of the diagonal
                            const uint64_t ad = smem_desc(sa + (uint32_t)t * a_bytes + (uint32_t)kk * 2u * OZ_CHUNK_BYTES,
                                                          OZ_CHUNK_BYTES, 128);
                            const uint64_t bd = smem_desc(sb + (uint32_t)(d - t) * b_bytes + (uint32_t)kk * OZ_CHUNK_BYTES,
                                                          OZ_CHUNK_BYTES / 2, 128);
                            wgmma_s8_m64n64k32(acc[j], ad, bd, (ks | kk | t) ? 1u : 0u);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
                mbar_arrive(&empty_bar[slot]);                        // this thread has finished reading the slot
            }
            if (!ok) break;
            // epilogue of the pass: Horner sum of the diagonals in FP64 (weight of the pass 2^(-12 - 7 d_lo)), row and
            // column scales, C (+)= result
            const long long te = clock64();
            const int npd = d_hi - d_lo + 1;
            const double wpass = __longlong_as_double((long long)(1023 - 12 - 7 * d_lo) << 52);
            const bool add = (g != npass - 1) || p.accumulate;
            const int row0 = mt * OZ_TILE + cw * 64 + wl * 16 + (lane >> 2);
            const double sa_r[2] = {p.sA[row0], p.sA[row0 + 8]};     // sA / sB are padded to whole 128-row tiles
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = nt * OZ_TN + 8 * j + 2 * (lane & 3) + e;
                    if (col >= p.N) continue;
                    const double wsb = wpass * p.sB[col];
#pragma unroll
                    for (int hr = 0; hr < 2; ++hr) {
                        const int row = row0 + 8 * hr;
                        if (row >= p.M) continue;
                        const int i = 4 * j + 2 * hr + e;
                        double h = 0.0;
#pragma unroll
                        for (int q = 3; q >= 0; --q)
                            if (q < npd) h = (q == npd - 1) ? oz_i2d(acc[q][i]) : fma(h, 0.0078125, oz_i2d(acc[q][i]));
                        h *= sa_r[hr];
                        double *cp = p.C + (int64_t)row * p.ldc + col;
                        *cp = add ? fma(h, wsb, *cp) : h * wsb;
                    }
                }
            }
            t_epi += clock64() - te;
        }
    }
    if (p.dbg && blockIdx.x == 0 && threadIdx.x == 128) {
        p.dbg[2] = clock64() - t0;
        p.dbg[3] = t_full;
        p.dbg[4] = t_epi;
    }
}

const bool g_split_fused = getenv("B200_OZ_SPLIT2") == nullptr;   // B200_OZ_SPLIT2=1: the two-pass split kernels (A/B)
int *g_abort_flag = nullptr;   // device int: raised by a wait that timed out (never in a correct run)
int g_abort_dev = -1;

int ensure_abort_flag() {
    int dev = 0;
    B200_CUDA_CHECK(cudaGetDevice(&dev));
    if (g_abort_flag == nullptr || dev != g_abort_dev) {
        B200_CUDA_CHECK(cudaMalloc(&g_abort_flag, sizeof(int)));
        B200_CUDA_CHECK(cudaMemset(g_abort_flag, 0, sizeof(int)));
        g_abort_dev = dev;
    }
    return B200_OK;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_ozaki_split_worksize(int64_t rows, int64_t k, int32_t slices) {
    if (rows <= 0 || k <= 0 || slices < 1 || slices > OZ_MAX_SLICES) return 0;
    return split_layout(rows, k, slices).total;
}

extern "C" int b200_ozaki_split_f64(int64_t rows, int64_t k, const double *X, int64_t ld_row, int64_t ld_k,
                                    int32_t slices, void *out_dev, int64_t out_bytes, b200_stream_t stream) {
    if (rows <= 0 || k <= 0) return set_error(B200_ERR_ARG, "ozaki_split: empty operand");
    if (slices < 1 || slices > OZ_MAX_SLICES) return set_error(B200_ERR_ARG, "ozaki_split: slices must be 1..%d", OZ_MAX_SLICES);
    if (ld_row != 1 && ld_k != 1) return set_error(B200_ERR_ARG, "ozaki_split: one of ld_row, ld_k must be 1");
    SplitLayout L = split_layout(rows, k, slices);
    if (out_bytes < L.total) return set_error(B200_ERR_ARG, "ozaki_split: output buffer too small (%lld < %lld)",
                                              (long long)out_bytes, (long long)L.total);
    if (L.kc > 65535) return set_error(B200_ERR_ARG, "ozaki_split: k too large");
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t *base = static_cast<uint8_t *>(out_dev);
    double *scale = reinterpret_cast<double *>(base + L.scale_off);
    unsigned long long *maxbits = reinterpret_cast<unsigned long long *>(base + L.max_off);
    if (slices <= OZ_FUSED_MAX_SLICES && g_split_fused) {
        const unsigned nblk = (unsigned)(L.rt * OZ_TILE / OZF_ROWS);
        if (ld_k == 1)
            oz_split_fused_kernel<true><<<nblk, OZF_THREADS, 0, st>>>(X, rows, k, ld_row, slices, L.rt, L.kc, scale, base);
        else
            oz_split_fused_kernel<false><<<nblk, OZF_THREADS, 0, st>>>(X, rows, k, ld_k, slices, L.rt, L.kc, scale, base);
        B200_CHECK_LAUNCH();
        return B200_OK;
    }
    if (ld_k == 1) {
        int rows_per_block = 8;
        oz_rowmax_kcontig_kernel<<<(unsigned)((rows + rows_per_block - 1) / rows_per_block), 32 * rows_per_block, 0, st>>>(
            X, rows, k, ld_row, maxbits);
        B200_CHECK_LAUNCH();
    } else {
        B200_CUDA_CHECK(cudaMemsetAsync(maxbits, 0, (size_t)L.rt * OZ_TILE * 8, st));
        int64_t ksplit = std::max<int64_t>(1, std::min<int64_t>((k + 255) / 256, 64));
        int64_t k_per_block = (k + ksplit - 1) / ksplit;
        dim3 grid((unsigned)((rows + 31) / 32), (unsigned)ksplit);
        oz_rowmax_rcontig_kernel<<<grid, 256, 0, st>>>(X, rows, k, ld_k, k_per_block, maxbits);
        B200_CHECK_LAUNCH();
    }
    dim3 grid((unsigned)((L.rt * OZ_TILE + 127) / 128), (unsigned)L.kc);
    oz_split_kernel<<<grid, 128, 0, st>>>(X, rows, k, ld_row, ld_k, slices, L.rt, L.kc, maxbits, scale, base);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

extern "C" int b200_ozaki_mm_f64(int64_t m, int64_t n, int64_t k, int32_t slices, const void *a_split,
                                 const void *b_split, double *C, int64_t ldc, int32_t accumulate,
                                 b200_stream_t stream) {
    if (m <= 0 || n <= 0 || k <= 0) return set_error(B200_ERR_ARG, "ozaki_mm: empty product");
    if (slices < 1 || slices > OZ_MAX_SLICES) return set_error(B200_ERR_ARG, "ozaki_mm: slices must be 1..%d", OZ_MAX_SLICES);
    // exactness of the int32 accumulation: k * 2^12 * (terms per diagonal) < 2^31
    if ((double)oz_k_chunks(k) * 16.0 * 4096.0 * slices >= 2147483648.0)
        return set_error(B200_ERR_ARG, "ozaki_mm: k = %lld too large for exact int32 accumulation with %d slices",
                         (long long)k, slices);
    int rc = ensure_abort_flag();
    if (rc) return rc;
    SplitLayout La = split_layout(m, k, slices), Lb = split_layout(n, k, slices);
    OzGemmArgs p;
    p.As = static_cast<const uint8_t *>(a_split);
    p.Bs = static_cast<const uint8_t *>(b_split);
    p.sA = reinterpret_cast<const double *>(p.As + La.scale_off);
    p.sB = reinterpret_cast<const double *>(p.Bs + Lb.scale_off);
    p.C = C;
    p.ldc = ldc;
    p.M = (int32_t)m;
    p.N = (int32_t)n;
    p.kc = (int32_t)La.kc;
    p.rta = (int32_t)La.rt;
    p.rtb = (int32_t)Lb.rt;
    p.slices = slices;
    p.accumulate = accumulate ? 1 : 0;
    p.abort_flag = g_abort_flag;
    p.dbg = nullptr;
    static const bool debug = getenv("B200_OZ_DEBUG") != nullptr;   // cycle counters of CTA 0 -> stderr (synchronises)
    long long *dbg_dev = nullptr;
    if (debug) {
        B200_CUDA_CHECK(cudaMalloc(&dbg_dev, 8 * sizeof(long long)));
        B200_CUDA_CHECK(cudaMemset(dbg_dev, 0, 8 * sizeof(long long)));
        p.dbg = dbg_dev;
    }
    // pipeline shape: as many k chunks per stage as leave at least two stages in shared memory
    static const int force_cps = getenv("B200_OZ_CPS") ? atoi(getenv("B200_OZ_CPS")) : 0;   // tuning knob (2 or 4)
    p.cps = force_cps == 2 ? 2 : 4;
    // a stage holds, per slice, the A tile (128 rows) and one half of the B tile (64 rows) of cps k chunks
    int64_t stage = 3LL * slices * p.cps * (OZ_CHUNK_BYTES / 2);
    if (OZ_SMEM_BUDGET / stage < 2) {
        p.cps = 2;
        stage = 3LL * slices * p.cps * (OZ_CHUNK_BYTES / 2);
    }
    p.nstages = (int32_t)std::min<int64_t>(OZ_MAX_STAGES, OZ_SMEM_BUDGET / stage);
    if (p.nstages < 1) return set_error(B200_ERR_ARG, "ozaki_mm: too many slices for shared memory");
    size_t smem = (size_t)p.nstages * stage;
    static bool attr_set = false;
    if (!attr_set) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(oz_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, OZ_SMEM_BUDGET));
        attr_set = true;
    }
    int64_t ntiles = oz_row_tiles(m) * ((n + OZ_TN - 1) / OZ_TN);
    int grid = (int)std::min<int64_t>(ntiles, sm_count());
    oz_gemm_kernel<<<grid, OZ_THREADS, smem, (cudaStream_t)stream>>>(p);
    B200_CHECK_LAUNCH();
    if (debug) {
        long long h[8];
        B200_CUDA_CHECK(cudaMemcpy(h, dbg_dev, sizeof(h), cudaMemcpyDeviceToHost));
        cudaFree(dbg_dev);
        fprintf(stderr, "[oz_gemm m=%lld n=%lld k=%lld s=%d cps=%d stages=%d] CTA0 cycles: producer total %lld wait_empty %lld | "
                "consumer total %lld wait_full %lld epilogue %lld\n",
                (long long)m, (long long)n, (long long)k, slices, p.cps, p.nstages, h[0], h[1], h[2], h[3], h[4]);
    }
    return B200_OK;
}

extern "C" int b200_ozaki_check_abort(void) {
    if (!g_abort_flag) return B200_OK;
    int flag = 0;
    B200_CUDA_CHECK(cudaMemcpy(&flag, g_abort_flag, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) {
        cudaMemset(g_abort_flag, 0, sizeof(int));
        return set_error(B200_ERR_CUDA, "ozaki kernel: a pipeline wait timed out (watchdog)");
    }
    return B200_OK;
}

extern "C" int64_t b200_ozaki_gemm_worksize(int64_t m, int64_t n, int64_t k, int32_t slices) {
    return b200_ozaki_split_worksize(m, k, slices) + 256 + b200_ozaki_split_worksize(n, k, slices);
}

extern "C" int b200_ozaki_gemm_f64(int64_t m, int64_t n, int64_t k, const double *A, int64_t lda, const double *B,
                                   int64_t ldb, double *C, int64_t ldc, int32_t slices, int32_t accumulate,
                                   void *work_dev, int64_t work_bytes, b200_stream_t stream) {
    int64_t wa = b200_ozaki_split_worksize(m, k, slices), wb = b200_ozaki_split_worksize(n, k, slices);
    if (wa == 0 || wb == 0) return set_error(B200_ERR_ARG, "ozaki_gemm: bad shape or slice count");
    int64_t off_b = (wa + 255) / 256 * 256;
    if (work_bytes < off_b + wb) return set_error(B200_ERR_ARG, "ozaki_gemm: workspace too small");
    uint8_t *w = static_cast<uint8_t *>(work_dev);
    int rc = b200_ozaki_split_f64(m, k, A, lda, 1, slices, w, wa, stream);
    if (rc) return rc;
    rc = b200_ozaki_split_f64(n, k, B, 1, ldb, slices, w + off_b, wb, stream);
    if (rc) return rc;
    return b200_ozaki_mm_f64(m, n, k, slices, w, w + off_b, C, ldc, accumulate, stream);
}
