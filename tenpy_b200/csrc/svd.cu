// svd.cu -- batched block-diagonal SVD and symmetric eigen-decomposition by one-sided block Jacobi.
//
// Replaces, on the GPU, the per-charge-block LAPACK calls of the reference:
//   npc._svd_worker (tenpy/linalg/np_conserved.py:4950) -> svd_robust.svd (svd_robust.py:37, gesdd/gesvd)
//   npc._eig_worker (np_conserved.py:5041)              -> np.linalg.eigh (syevd; zheevd for complex Hermitian blocks)
//
// Algorithm (all blocks of one Array in one batch):
//   Each matrix is held as Y (q x p, q <= p, row-major, rows = the vectors to orthogonalise; Y = A or A^T)
//   plus W (q x q) = accumulated orthogonal row transformation, W Y0 = Y.  Rows are grouped in blocks of
//   JB = 16.  One Jacobi *round* processes nb/2 disjoint block pairs (round-robin tournament); one CTA
//   owns one pair = a 32-row panel P:
//     1. G = P P^T (32x32) streamed through shared memory with FP64 tensor-core MMAs,
//     2. G = Q L Q^T by a parallel cyclic two-sided Jacobi in shared memory,
//     3. P <- Q^T P and the same rows of W <- Q^T W (second streamed pass, DMMA).
//   A pair whose scaled off-diagonal max |g_ij|/sqrt(g_ii g_jj) is below tol is left untouched; a matrix
//   is converged once a full cycle of rounds touched nothing.  Singular values = row norms of Y,
//   sorted on the host (k doubles), vectors written by a final gather kernel.
// Complex blocks (b200_block_svd_z) run the same driver and the same round kernels instantiated with CPLX = true: Y and
// W get planar imaginary parts, G = P P^H is Hermitian and the transformation unitary (see jacobi_eig_kernel).
// Never produces NaN for finite input (the reference falls back gesdd->gesvd for that, npc:4971-4978).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <initializer_list>
#include <limits>
#include <numeric>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "scaling.cuh"

namespace b200 {

constexpr int JB = 16;          // rows per block
constexpr int JP = 2 * JB;      // rows per panel
constexpr int JKC = 128;        // streamed chunk (columns)
constexpr int JLDP = JKC + 4;   // smem row stride of a panel chunk
constexpr int JTHREADS = 256;
constexpr int JLDG = JP + 1;
constexpr int J_NSPLIT_MAX = 16;    // column splits of the streaming phases of one pair
constexpr int J_INNER_SWEEPS = 2;   // the pivot block only has to be diagonalised "well enough" per round: the outer sweep
                                    // count is the same for 2 and 4 (profiles/jacobi_sweeps_study.md; 4 until round 1)

struct JMat {
    int64_t y_off, w_off, snorm_off;       // element offsets into the f64 work area
    int64_t prep_off;                      // m + n doubles: squared row / column norms of A (orientation, pre-sort)
    int64_t a_off, u_off, s_off, vt_off;   // element offsets into the caller's buffers
    int32_t m, n;                          // original shape
    int32_t q, p;                          // vectors, vector length
    int32_t qp, nb;                        // padded vector count (= nb*JB), number of row blocks (even)
    int32_t ldy, ldw;
    int32_t transposed;                    // Y = A^T
    int32_t cta_begin;                     // first CTA of this matrix in a round launch
    int32_t perm_off;                      // offset into the int32 permutation pool
    int32_t nb_act;                        // active row blocks (even, >= 2): logical rows [0, nb_act*JB)
    int32_t rmap_off;                      // offset into the int32 row-map pool (logical row -> physical row)
    int32_t n_act;                         // number of non-deflated vectors
    double defl;                           // deflation threshold: rows with norm <= defl are negligible
    double shift;                          // eigh: diagonal shift
    int64_t yi_off, wi_off;                // complex SVD: imaginary parts of Y and W (planar; y_off / w_off = real parts)
    double scale;                          // Y = scale * A, scale = pow2_scale(max |a_ij|) (exact); S, W = norms / scale
    int32_t cplx, pad_;                    // 1: complex matrix (b200_block_svd_z)
    double amax;                           // max |a_ij| (jacobi_amax_kernel; 0 before it runs)
};

// active row blocks for n_act active vectors: an even number (the round-robin pairs the blocks), at least 2, at most nb
__host__ __device__ inline int j_nb_act(int n_act, int nb) {
    int nb_act = (n_act + JB - 1) / JB;
    if (nb_act < 2) nb_act = 2;
    if (nb_act & 1) ++nb_act;
    return nb_act > nb ? nb : nb_act;
}

// dynamic shared memory of the streaming phases: two pipeline stages of one panel chunk per plane
template <bool CPLX>
constexpr int jacobi_smem_bytes() { return 2 * (CPLX ? 2 : 1) * JP * JLDP * (int)sizeof(double); }

// Gram diagonals at or below J_GRAM_MIN (Y is the scaled block, max |y| in [1, 2)) are lost in the absolute rounding of
// subnormal products (~p 2^-1075 per entry): such rows cannot be resolved and are inert, like deflated ones.  Far below
// any deflation threshold, so this only decides anything with deflation off, for rows graded below ~1e-149.
constexpr double J_GRAM_MIN = 0x1p-990;
__device__ __forceinline__ bool j_normal(double x) { return x >= 2.2250738585072014e-308 && x <= 1.7976931348623157e308; }
// sqrt(a b) for a, b >= 0 without under- or overflow of the product.  Where the product is normal this is the plain
// sqrt(a * b), so every decision on normal-range data is the one it always was.
__device__ __forceinline__ double j_sqrt_prod(double a, double b) {
    const double d = a * b;
    return j_normal(d) ? sqrt(d) : sqrt(a) * sqrt(b);
}

// max of v over the CTA (JTHREADS threads; red: 32 doubles of shared memory), returned to every thread
__device__ __forceinline__ double j_cta_max(double v, double *red, int lane, int warp) {
    v = warp_max(v);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = 0.0;
#pragma unroll
    for (int w = 0; w < JTHREADS / 32; ++w) v = fmax(v, red[w]);
    return v;
}

// rank of row i of a pivot block (sA: its Gram matrix, stride JLDG) when the rows are ordered by descending diagonal
// (eigenvalue = norm^2), ties by index.  The key is clamped at 0: the rotated diagonal of a row at rounding level can come
// out slightly negative and must not sort behind the all-zero padding rows (q..qp-1, always the last positions of a pair),
// or the padding content (zero Y, W = a unit vector outside the block) would move into a real row
__device__ __forceinline__ int j_row_rank(const double *sA, int i) {
    const double di = fmax(sA[i * JLDG + i], 0.0);
    int rk = 0;
    for (int k = 0; k < JP; ++k) {
        const double dk = fmax(sA[k * JLDG + k], 0.0);
        if (dk > di || (dk == di && k < i)) ++rk;
    }
    return rk;
}

__device__ __forceinline__ void j_load_chunk(double *sP, const double *base, int ld, const int *prow, int col0,
                                             int tid) {
    constexpr int CH = JP * (JKC / 2);
#pragma unroll
    for (int c = tid; c < CH; c += JTHREADS) {
        int r = c / (JKC / 2), cc = (c % (JKC / 2)) * 2;
        int grow = prow[r];
        int gcol = col0 + cc;
        bool ok = gcol < ld;
        const double *src = ok ? base + (int64_t)grow * ld + gcol : base;
        cp_async16(sP + r * JLDP + cc, src, ok ? 16 : 0);
    }
}

// rows of `base` (ld) <- Q^T rows for the column chunks ch0, ch0+chstep, ... ; prow[0..31] = physical rows.
// q[0] = fragments of Q^T; CPLX: q[1] = those of its imaginary part, basei = the imaginary plane of `base`
template <bool CPLX>
__device__ __forceinline__ void j_apply(double *bufs, const double (&q)[CPLX ? 2 : 1][2][4][4], double *base,
                                        double *basei, int ld, const int *prow, int tid, int ch0, int chstep) {
    constexpr int STAGE = (CPLX ? 2 : 1) * JP * JLDP;
    const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int nch = (ld + JKC - 1) / JKC;
    if (ch0 >= nch) return;
    j_load_chunk(bufs, base, ld, prow, ch0 * JKC, tid);
    if constexpr (CPLX) j_load_chunk(bufs + JP * JLDP, basei, ld, prow, ch0 * JKC, tid);
    cp_async_commit();
    int it = 0;
    for (int ch = ch0; ch < nch; ch += chstep, ++it) {
        if (ch + chstep < nch) {
            double *nxt = bufs + ((it + 1) & 1) * STAGE;
            j_load_chunk(nxt, base, ld, prow, (ch + chstep) * JKC, tid);
            if constexpr (CPLX) j_load_chunk(nxt + JP * JLDP, basei, ld, prow, (ch + chstep) * JKC, tid);
        }
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        const double *sr = bufs + (it & 1) * STAGE, *si = sr + JP * JLDP;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int nt = warp * 2 + h;
            const int col = ch * JKC + nt * 8;
            if (col < ld) {
                double acc[2][4], acci[2][4];
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc[i][e] = acci[i][e] = 0.0;
#pragma unroll
                for (int k8 = 0; k8 < 4; ++k8) {
                    const int b0 = (k8 * 8 + t) * JLDP + nt * 8 + g, b1 = (k8 * 8 + t + 4) * JLDP + nt * 8 + g;
                    double br[2] = {sr[b0], sr[b1]};
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        dmma_16x8x8(acc[i], q[0][i][k8], br);
                        if constexpr (CPLX) {   // Re += -Qi Pi,  Im += Qr Pi + Qi Pr
                            const double(&qi)[4] = q[1][i][k8];
                            double nqi[4] = {-qi[0], -qi[1], -qi[2], -qi[3]};
                            double bi[2] = {si[b0], si[b1]};
                            dmma_16x8x8(acc[i], nqi, bi);
                            dmma_16x8x8(acci[i], q[0][i][k8], bi);
                            dmma_16x8x8(acci[i], qi, br);
                        }
                    }
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int64_t o = (int64_t)prow[i * 16 + g + 8 * hh] * ld + col + 2 * t;
                        *reinterpret_cast<double2 *>(base + o) = make_double2(acc[i][2 * hh], acc[i][2 * hh + 1]);
                        if constexpr (CPLX)
                            *reinterpret_cast<double2 *>(basei + o) = make_double2(acci[i][2 * hh], acci[i][2 * hh + 1]);
                    }
                }
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
}

// the 32 physical rows of pair `j` of matrix `mt` in round `round` (round-robin tournament over the active
// blocks); returns false if this CTA has no pair.  Must be followed by __syncthreads().
__device__ __forceinline__ bool j_pair_rows(const JMat &mt, int j, int round, const int *__restrict__ rmap,
                                            int *s_rows, int tid) {
    const int nb = mt.nb_act;   // deflated (negligible) rows live in the blocks >= nb_act and are never touched
    if (2 * j >= nb) return false;
    int ba, bb;
    const int nr = nb - 1;
    const int r = round % nr;
    if (j == 0) {
        ba = nb - 1;
        bb = r;
    } else {
        ba = (r + j) % nr;
        bb = (r - j + nr) % nr;
    }
    if (ba > bb) {
        int tmp = ba;
        ba = bb;
        bb = tmp;
    }
    if (tid < JP) s_rows[tid] = rmap[mt.rmap_off + (tid < JB ? ba * JB + tid : bb * JB + tid - JB)];
    return true;
}

// One Jacobi round = three launches, so that the streaming phases use the whole GPU:
//   jacobi_gram_kernel  grid (nsplit, pairs): partial G = P P^T over a subset of the column chunks (DMMA),
//                       one 32x32 partial per split in Gbuf[pair][split]
//   jacobi_eig_kernel   grid (pairs): convergence test, parallel cyclic Jacobi on G, Q^T (rows ordered by descending
//   (or _v3)            eigenvalue) -> QTbuf[pair], flag[pair] = rotated
//   jacobi_apply_kernel grid (nsplit, pairs, 2): P <- Q^T P (z = 0) and the same rows of W <- Q^T W (z = 1)
// CPLX = true (complex blocks): every streamed chunk has a real and an imaginary plane, each phase is four real DMMA
// products (Re G = Pr Pr^T + Pi Pi^T, Im G = Pi Pr^T - Pr Pi^T;  Re P' = Tr Pr - Ti Pi, Im P' = Tr Pi + Ti Pr), and the Gram
// partials and Q^T (= T) are stored as [real 32x32 | imaginary 32x32] per pair (and split).
// (the three phases are device functions so that jacobi_round_fused_kernel can run them back to back in one launch; buffers
// one phase writes and the next one reads -- Gbuf, QTbuf, flags, work -- are deliberately NOT const __restrict__ there: the
// read-only data path is not coherent with writes of the same kernel)
template <bool CPLX>
__device__ __forceinline__ void jacobi_gram_body(double *bufs, const double *work, const JMat *__restrict__ mats,
                                                 const int *__restrict__ cta_mat, const int *__restrict__ rmap, int round,
                                                 const int *__restrict__ done, double *Gbuf, int split, int nsplit, int pair) {
    constexpr int NPL = CPLX ? 2 : 1, STAGE = NPL * JP * JLDP;
    __shared__ int s_rows[JP];
    const int mi = cta_mat[pair];
    if (done[mi]) return;
    const JMat mt = mats[mi];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    if (!j_pair_rows(mt, pair - mt.cta_begin, round, rmap, s_rows, tid)) return;
    __syncthreads();
    const double *Y = work + mt.y_off, *Yi = work + mt.yi_off;
    const int ld = mt.ldy;
    const int nch = (ld + JKC - 1) / JKC;
    const int ch0 = split, chstep = nsplit;
    if (ch0 >= nch) return;
    const int tm = warp >> 2, tn = warp & 3;  // 2 x 4 tiles of 16 x 8
    double acc[4] = {0.0, 0.0, 0.0, 0.0}, acci[4] = {0.0, 0.0, 0.0, 0.0};
    j_load_chunk(bufs, Y, ld, s_rows, ch0 * JKC, tid);
    if constexpr (CPLX) j_load_chunk(bufs + JP * JLDP, Yi, ld, s_rows, ch0 * JKC, tid);
    cp_async_commit();
    int it = 0;
    for (int ch = ch0; ch < nch; ch += chstep, ++it) {
        if (ch + chstep < nch) {
            double *nxt = bufs + ((it + 1) & 1) * STAGE;
            j_load_chunk(nxt, Y, ld, s_rows, (ch + chstep) * JKC, tid);
            if constexpr (CPLX) j_load_chunk(nxt + JP * JLDP, Yi, ld, s_rows, (ch + chstep) * JKC, tid);
        }
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        const double *sr = bufs + (it & 1) * STAGE, *si = sr + JP * JLDP;
#pragma unroll (CPLX ? 4 : JKC / 8)
        for (int k8 = 0; k8 < JKC / 8; ++k8) {
            const int ao = (tm * 16 + g) * JLDP + k8 * 8 + t, bo = (tn * 8 + g) * JLDP + k8 * 8 + t;
            double ar[4] = {sr[ao], sr[ao + 8 * JLDP], sr[ao + 4], sr[ao + 8 * JLDP + 4]};
            double br[2] = {sr[bo], sr[bo + 4]};
            dmma_16x8x8(acc, ar, br);
            if constexpr (CPLX) {   // Re G += Pi Pi^T,  Im G += Pi Pr^T - Pr Pi^T
                double ai[4] = {si[ao], si[ao + 8 * JLDP], si[ao + 4], si[ao + 8 * JLDP + 4]};
                double nar[4] = {-ar[0], -ar[1], -ar[2], -ar[3]};
                double bi[2] = {si[bo], si[bo + 4]};
                dmma_16x8x8(acc, ai, bi);
                dmma_16x8x8(acci, ai, br);
                dmma_16x8x8(acci, nar, bi);
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
    // partial result of this column split (summed in a fixed order by the eigen-solver phase: deterministic)
    double *G = Gbuf + ((int64_t)pair * nsplit + split) * (NPL * JP * JP);
    const int r0 = tm * 16 + g, c0 = tn * 8 + 2 * t;
#pragma unroll
    for (int part = 0; part < NPL; ++part) {
        const double *a = part ? acci : acc;
        double *Gp = G + part * (JP * JP);
        Gp[r0 * JP + c0] = a[0];
        Gp[r0 * JP + c0 + 1] = a[1];
        Gp[(r0 + 8) * JP + c0] = a[2];
        Gp[(r0 + 8) * JP + c0 + 1] = a[3];
    }
}

template <bool CPLX>
__global__ void __launch_bounds__(JTHREADS)
    jacobi_gram_kernel(const double *__restrict__ work, const JMat *__restrict__ mats, const int *__restrict__ cta_mat,
                       const int *__restrict__ rmap, int round, const int *__restrict__ done,
                       double *__restrict__ Gbuf) {
    extern __shared__ __align__(16) double jsmem[];
    jacobi_gram_body<CPLX>(jsmem, work, mats, cta_mat, rmap, round, done, Gbuf, blockIdx.x, gridDim.x, blockIdx.y);
}

// Pivot solver 1, real (CPLX = false) and complex: grid (pairs), G and T in shared memory.  Convergence test, then T with
// T G T^H diagonal by parallel cyclic Jacobi (16 disjoint pairs per rotation set, round-robin order), rows of T ordered by
// descending eigenvalue -> QTbuf[pair], flag[pair] = rotated.  The rotation of the pair (p, q) is the real rotation (c, s)
// of (g_pp, g_qq, |g_pq|) after the phase e = g_pq / |g_pq| of a complex g_pq is stripped (e = 1 for real blocks):
//   rows of G and T:  row p <- c x_p - s e x_q,  row q <- s x_p + c e x_q
//   columns of G:     col p <- c y_p - s conj(e) y_q,  col q <- s y_p + c conj(e) y_q
template <bool CPLX>
__global__ void __launch_bounds__(JTHREADS)
    jacobi_eig_kernel(const JMat *__restrict__ mats, const int *__restrict__ cta_mat, int *__restrict__ rot_count,
                      const int *__restrict__ done, double tol_scale, const double *__restrict__ Gbuf, int nsplit,
                      double *__restrict__ QTbuf, int *__restrict__ flags, int inner_sweeps) {
    constexpr int NPL = CPLX ? 2 : 1;
    __shared__ double sG[NPL][JP * JLDG], sT[NPL][JP * JLDG];   // [real | imaginary]
    __shared__ double cs_c[JB], cs_s[JB], cs_er[JB], cs_ei[JB];
    __shared__ int pr_p[JB], pr_q[JB];
    __shared__ double red[32];
    __shared__ int s_rank[JP];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) flags[blockIdx.x] = 0;
    const int mi = cta_mat[blockIdx.x];
    if (done[mi]) return;
    const JMat mt = mats[mi];
    if (2 * (blockIdx.x - mt.cta_begin) >= mt.nb_act) return;
    {
        const int nch = (mt.ldy + JKC - 1) / JKC;
        const int ns = nsplit < nch ? nsplit : nch;
        const double *G = Gbuf + (int64_t)blockIdx.x * nsplit * (NPL * JP * JP);
        for (int idx = tid; idx < JP * JP; idx += JTHREADS) {
            const int r = idx / JP, c = idx % JP;
#pragma unroll
            for (int pl = 0; pl < NPL; ++pl) {
                double v = 0.0;
                for (int sp = 0; sp < ns; ++sp) v += G[sp * (NPL * JP * JP) + pl * (JP * JP) + idx];
                sG[pl][r * JLDG + c] = v;
                sT[pl][r * JLDG + c] = (pl == 0 && r == c) ? 1.0 : 0.0;
            }
        }
    }
    __syncthreads();

    // ---- convergence measure of this pair: max |g_rc| / sqrt(g_rr g_cc) over the non-negligible rows ----
    // (square roots taken separately where g_rr g_cc over- or underflows: blocks scaled near 1e+-150)
    const double defl2 = fmax(mt.defl * mt.defl, J_GRAM_MIN);
    double offmax = 0.0;
    for (int idx = tid; idx < JP * JP; idx += JTHREADS) {
        const int r = idx / JP, c = idx % JP;
        if (r < c) {
            const double drr = sG[0][r * JLDG + r], dcc = sG[0][c * JLDG + c];
            if (drr > defl2 && dcc > defl2) {   // negligible (deflated) rows are inert
                if constexpr (CPLX)
                    offmax = fmax(offmax, hypot(sG[0][r * JLDG + c], sG[1][r * JLDG + c]) / (sqrt(drr) * sqrt(dcc)));
                else
                    offmax = fmax(offmax, fabs(sG[0][r * JLDG + c]) / j_sqrt_prod(drr, dcc));
            }
        }
    }
    offmax = j_cta_max(offmax, red, lane, warp);
    const double tol = tol_scale * sqrt((double)mt.p);
    if (!(offmax > tol)) return;  // uniform for the whole CTA
    if (tid == 0) atomicAdd(&rot_count[mi], 1);

    const double tol_in = 1e-15;
    for (int sweep = 0; sweep < inner_sweeps; ++sweep) {
        int any = 0;
        for (int step = 0; step < JP - 1; ++step) {
            if (tid < JB) {
                int a, b;
                if (tid == 0) {
                    a = JP - 1;
                    b = step;
                } else {
                    a = (step + tid) % (JP - 1);
                    b = (step - tid + (JP - 1)) % (JP - 1);
                }
                const int p = a < b ? a : b, q = a < b ? b : a;
                const double gpp = sG[0][p * JLDG + p], gqq = sG[0][q * JLDG + q], gpq = sG[0][p * JLDG + q];
                double c = 1.0, s = 0.0, er = 1.0, ei = 0.0;
                // t = tan(theta) of the Jacobi rotation: one sqrt or hypot, one division, one rsqrt
                if constexpr (CPLX) {
                    const double gi = sG[1][p * JLDG + q], ag = hypot(gpq, gi);
                    if (gpp > defl2 && gqq > defl2 && ag > tol_in * sqrt(gpp) * sqrt(gqq)) {
                        er = gpq / ag;
                        ei = gi / ag;
                        const double aa = gqq - gpp, bb = 2.0 * ag;
                        const double hh = hypot(aa, bb);
                        const double tt = (aa >= 0.0) ? bb / (aa + hh) : bb / (aa - hh);
                        c = rsqrt(1.0 + tt * tt);
                        s = tt * c;
                        any = 1;
                    }
                } else {   // (hypot only where aa^2 + bb^2 is not a normal number)
                    const double lim = tol_in * j_sqrt_prod(fabs(gpp), fabs(gqq));
                    if (fabs(gpq) > lim && gpp > defl2 && gqq > defl2) {
                        const double aa = gqq - gpp, bb = 2.0 * gpq;
                        const double h2 = aa * aa + bb * bb;
                        const double hh = j_normal(h2) ? sqrt(h2) : hypot(aa, bb);
                        const double tt = (aa >= 0.0) ? bb / (aa + hh) : bb / (aa - hh);
                        c = rsqrt(1.0 + tt * tt);
                        s = tt * c;
                        any = 1;
                    }
                }
                pr_p[tid] = p;
                pr_q[tid] = q;
                cs_c[tid] = c;
                cs_s[tid] = s;
                if constexpr (CPLX) {
                    cs_er[tid] = er;
                    cs_ei[tid] = ei;
                }
            }
            __syncthreads();
            // rows of G and T:  row p <- c x_p - s y,  row q <- s x_p + c y,  y = e x_q
            for (int idx = tid; idx < JB * JP; idx += JTHREADS) {
                const int jj = idx / JP, col = idx % JP;
                const int p = pr_p[jj], q = pr_q[jj];
                const double c = cs_c[jj], s = cs_s[jj];
#pragma unroll
                for (int which = 0; which < 2; ++which) {
                    double *Xr = which ? sT[0] : sG[0];
                    const double xpr = Xr[p * JLDG + col];
                    double yr = Xr[q * JLDG + col];
                    if constexpr (CPLX) {
                        double *Xi = which ? sT[1] : sG[1];
                        const double er = cs_er[jj], ei = cs_ei[jj];
                        const double xpi = Xi[p * JLDG + col], xqr = yr, xqi = Xi[q * JLDG + col];
                        yr = er * xqr - ei * xqi;
                        const double yi = er * xqi + ei * xqr;
                        Xi[p * JLDG + col] = c * xpi - s * yi;
                        Xi[q * JLDG + col] = s * xpi + c * yi;
                    }
                    Xr[p * JLDG + col] = c * xpr - s * yr;
                    Xr[q * JLDG + col] = s * xpr + c * yr;
                }
            }
            __syncthreads();
            // columns of G (G <- G T^H):  col p <- c y_p - s z,  col q <- s y_p + c z,  z = conj(e) y_q
            for (int idx = tid; idx < JB * JP; idx += JTHREADS) {
                const int jj = idx / JP, row = idx % JP;
                const int p = pr_p[jj], q = pr_q[jj];
                const double c = cs_c[jj], s = cs_s[jj];
                const double ypr = sG[0][row * JLDG + p];
                double zr = sG[0][row * JLDG + q];
                if constexpr (CPLX) {
                    const double er = cs_er[jj], ei = cs_ei[jj];
                    const double ypi = sG[1][row * JLDG + p], yqr = zr, yqi = sG[1][row * JLDG + q];
                    zr = er * yqr + ei * yqi;
                    const double zi = er * yqi - ei * yqr;
                    sG[1][row * JLDG + p] = c * ypi - s * zi;
                    sG[1][row * JLDG + q] = s * ypi + c * zi;
                }
                sG[0][row * JLDG + p] = c * ypr - s * zr;
                sG[0][row * JLDG + q] = s * ypr + c * zr;
            }
            __syncthreads();
        }
        if (!__syncthreads_or(any)) break;
    }
    // rows of T ordered by descending eigenvalue (norm^2): helps the outer convergence (de Rijk)
    if (tid < JP) s_rank[tid] = j_row_rank(sG[0], tid);
    __syncthreads();
    double *QT = QTbuf + (int64_t)blockIdx.x * (NPL * JP * JP);
    for (int idx = tid; idx < JP * JP; idx += JTHREADS) {
        const int i = idx / JP, k = idx % JP;
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) QT[pl * (JP * JP) + s_rank[i] * JP + k] = sT[pl][i * JLDG + k];
    }
    if (tid == 0) flags[blockIdx.x] = 1;
}

// Version 3 of the pivot eigen-solver: G and Q live in REGISTERS, rotations go through warp shuffles, shared memory is
// only the transposition buffer -> two barriers per rotation set and no dependent shared-memory read-modify-write chains
// (version 1: three barriers and three shared-memory passes per set).
//   thread (warp w, lane l) holds G[l][4w+i] and Q[4w+i][l], i < 4 (256 threads).
//   one rotation set (16 disjoint pairs (p, q), the same round-robin order as version 1):
//     1. every lane computes the rotation of the pair its row index l belongs to from sA (= the current G in shared
//        memory: G[p][p], G[q][q], G[p][q]); the 8 warps do this redundantly instead of waiting for one another;
//     2. rows:    G' = J G        lane l combines its value with lane partner(l)'s (shuffle);
//     3. columns: G'' = G' J^T    = (J G'^T)^T and G'' is symmetric: write G' to sT, barrier, read it TRANSPOSED and
//        apply the same row rotation again -- the result is G''[l][c] in the thread that holds G[l][c];
//     4. Q <- Q J^T (columns p, q of every row: lanes p, q of the same warp, shuffle);
//     5. write G'' to sA for the parameters of the next set, barrier.
// Same interface and the same rotations (to rounding) as version 1.
// Jacobi rotation (c, s) that annihilates g_pq:  t = tan(theta) = sign(z) / (|z| + sqrt(1 + z^2)),  z = (g_qq - g_pp) / (2 g_pq),
// c = 1 / sqrt(1 + t^2), s = t c  (the same rotation as version 1).  The double-precision sqrt / division / rsqrt of the
// straightforward formula are ~100-instruction dependent chains each and sit on the critical path of every rotation set;
// here each is a single-precision hardware approximation refined by two Newton steps in double precision (relative error
// ~1e-15; c^2 + s^2 = 1 to rounding by construction, so the transformation stays orthogonal whatever the error of t).
__device__ __forceinline__ double jeig3_rcp(double x) {          // 1/x for |x| in [1e-30, 1e30]
    double r = (double)__frcp_rn((float)x);
    r = fma(r, fma(-x, r, 1.0), r);
    return fma(r, fma(-x, r, 1.0), r);
}
__device__ __forceinline__ double jeig3_rsqrt(double x) {        // 1/sqrt(x) for x in [1, 1e30]
    double r = (double)rsqrtf((float)x);
    r = r * fma(-0.5 * x, r * r, 1.5);
    return r * fma(-0.5 * x, r * r, 1.5);
}
__device__ __forceinline__ void jeig3_rotation(double gpp, double gqq, double gpq, double &c, double &s) {
    const double aa = gqq - gpp, bb = 2.0 * gpq;
    // bring bb to [1, 2) by a power of two (exact) so that the single-precision seed cannot over- or underflow
    int eb = (int)((__double_as_longlong(bb) >> 52) & 0x7ff);
    eb = min(max(eb, 2), 2044);
    const double scale = __longlong_as_double((long long)(2046 - eb) << 52);
    const double z = (aa * scale) * jeig3_rcp(bb * scale);
    const double az = fabs(z);
    double t;
    if (az < 1.e12) {
        const double y = fma(z, z, 1.0);
        const double den = az + y * jeig3_rsqrt(y);               // |z| + sqrt(1 + z^2), in [1, 2e12]
        t = copysign(jeig3_rcp(den), z);
    } else {
        t = 0.5 / z;                                              // also covers z = +-inf (t = 0)
    }
    c = jeig3_rsqrt(fma(t, t, 1.0));
    s = t * c;
}

__device__ __forceinline__ int jeig3_partner(int x, int step) {
    // round-robin tournament over JP = 32 indices, index 31 fixed: pairs (31, step) and ((step+j) % 31, (step-j) % 31)
    if (x == JP - 1) return step;
    int j = x - step;
    if (j < 0) j += JP - 1;
    if (j == 0) return JP - 1;
    int y = (j <= JB - 1) ? step - j : step + (JP - 1 - j);
    if (y < 0) y += JP - 1;
    if (y >= JP - 1) y -= JP - 1;
    return y;
}

__device__ __forceinline__ void jacobi_eig_v3_body(const JMat *__restrict__ mats, const int *__restrict__ cta_mat,
                                                   int *rot_count, const int *__restrict__ done, double tol_scale,
                                                   const double *Gbuf, int nsplit, double *QTbuf, int *flags, int inner_sweeps,
                                                   int round, int pair) {
    __shared__ double sA[JP * JLDG];
    __shared__ double sT[JP * JLDG];
    __shared__ double red[32];
    __shared__ int s_rank[JP];
    __shared__ int s_any;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) flags[pair] = 0;
    const int mi = cta_mat[pair];
    if (done[mi]) return;
    const JMat mt = mats[mi];
    if (2 * (pair - mt.cta_begin) >= mt.nb_act) return;
    double g[4], qv[4];
    {
        const int nch = (mt.ldy + JKC - 1) / JKC;
        const int ns = nsplit < nch ? nsplit : nch;
        const double *G = Gbuf + (int64_t)pair * nsplit * (JP * JP);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = 4 * warp + i;
            double v = 0.0;
#pragma unroll 4
            for (int sp = 0; sp < ns; ++sp) v += G[sp * (JP * JP) + c * JP + lane];   // G[c][l] = G[l][c], coalesced
            g[i] = v;
            sA[lane * JLDG + c] = v;
            qv[i] = (c == lane) ? 1.0 : 0.0;
        }
    }
    if (tid == 0) s_any = 0;
    __syncthreads();
    // ---- convergence measure of this pair (as version 1) ----
    const double defl2 = fmax(mt.defl * mt.defl, J_GRAM_MIN);
    double offmax = 0.0;
    {
        const double dl = sA[lane * JLDG + lane];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = 4 * warp + i;
            const double dc = sA[c * JLDG + c];
            if (lane < c && dl > defl2 && dc > defl2) offmax = fmax(offmax, fabs(g[i]) / j_sqrt_prod(dl, dc));
        }
    }
    offmax = j_cta_max(offmax, red, lane, warp);
    const double tol = tol_scale * sqrt((double)mt.p);
    if (!(offmax > tol)) return;  // uniform for the whole CTA
    if (tid == 0) atomicAdd(&rot_count[mi], 1);

    const double tol_in = 1e-15;
    // inner_sweeps == 0 ("cross" mode): one pass over the 16 x 16 pairs BETWEEN the two row blocks only (16 rotation sets
    // instead of 31 per pass); the pairs inside a block are rotated once per outer sweep, in the round in which every block
    // of the matrix is paired (round % (nb_act - 1) == 0: one full pass there).  Together: the cyclic element-wise Jacobi
    // sweep in block order, every pair of rows rotated exactly once per outer sweep.
    const int nr_blk = mt.nb_act - 1;
    const bool cross = inner_sweeps == 0 && nr_blk > 1 && (round % nr_blk) != 0;
    const int nsteps = cross ? JB : JP - 1;
    if (inner_sweeps == 0) inner_sweeps = 1;
    for (int sweep = 0; sweep < inner_sweeps; ++sweep) {
        for (int step = 0; step < nsteps; ++step) {
            // 1. rotation of the pair that contains row index `lane`
            const int partner = cross ? (lane < JB ? JB + ((lane + step) & (JB - 1)) : ((lane - JB - step) & (JB - 1)))
                                      : jeig3_partner(lane, step);
            const bool is_p = lane < partner;
            const int p = is_p ? lane : partner, q = is_p ? partner : lane;
            const double gpp = sA[p * JLDG + p], gqq = sA[q * JLDG + q], gpq = sA[p * JLDG + q];
            double c = 1.0, sn = 0.0;
            // |g_pq| > tol_in sqrt(g_pp g_qq), squared; with square roots taken separately where a product is not normal
            const double g2 = gpq * gpq, rhs = (tol_in * tol_in) * fabs(gpp * gqq);
            const bool off = (j_normal(g2) && j_normal(rhs)) ? g2 > rhs : fabs(gpq) > tol_in * j_sqrt_prod(fabs(gpp), fabs(gqq));
            if (off && gpp > defl2 && gqq > defl2) {
                jeig3_rotation(gpp, gqq, gpq, c, sn);
                if (warp == 0) s_any = 1;     // benign race: every writer stores 1
            }
            // row p: c x_p - s x_q ;  row q: s x_p + c x_q   -> as "own * c + other * (-s | +s)"
            const double so = is_p ? -sn : sn;
            // 2. rows of G
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double y = __shfl_sync(0xffffffffu, g[i], partner);
                g[i] = fma(so, y, c * g[i]);
                sT[lane * JLDG + 4 * warp + i] = g[i];
            }
            // 4. columns of Q (independent of the barrier below)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double y = __shfl_sync(0xffffffffu, qv[i], partner);
                qv[i] = fma(so, y, c * qv[i]);
            }
            __syncthreads();
            // 3. columns of G through the transposed read
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double t = sT[(4 * warp + i) * JLDG + lane];
                const double y = __shfl_sync(0xffffffffu, t, partner);
                g[i] = fma(so, y, c * t);
                sA[lane * JLDG + 4 * warp + i] = g[i];
            }
            __syncthreads();
        }
        const int any = s_any;
        __syncthreads();
        if (!any) break;
        if (tid == 0) s_any = 0;
        __syncthreads();
    }
    // order the new rows by descending eigenvalue (norm^2)
    if (tid < JP) s_rank[tid] = j_row_rank(sA, tid);
    __syncthreads();
    double *QT = QTbuf + (int64_t)pair * (JP * JP);
    // QT[rank[i]][k] = Q[k][i]; this thread holds Q[4w+j][lane]
#pragma unroll
    for (int i = 0; i < 4; ++i) QT[s_rank[lane] * JP + 4 * warp + i] = qv[i];
    if (tid == 0) flags[pair] = 1;
}

__global__ void __launch_bounds__(JTHREADS)
    jacobi_eig_kernel_v3(const JMat *__restrict__ mats, const int *__restrict__ cta_mat, int *__restrict__ rot_count,
                         const int *__restrict__ done, double tol_scale, const double *__restrict__ Gbuf, int nsplit,
                         double *__restrict__ QTbuf, int *__restrict__ flags, int inner_sweeps, int round) {
    jacobi_eig_v3_body(mats, cta_mat, rot_count, done, tol_scale, Gbuf, nsplit, QTbuf, flags, inner_sweeps, round, blockIdx.x);
}

template <bool CPLX>
__device__ __forceinline__ void jacobi_apply_body(double *bufs, double *work, const JMat *__restrict__ mats,
                                                  const int *__restrict__ cta_mat, const int *__restrict__ rmap, int round,
                                                  const double *QTbuf, const int *flags, int split, int nsplit, int pair,
                                                  int which) {
    constexpr int NPL = CPLX ? 2 : 1;
    __shared__ int s_rows[JP];
    if (!flags[pair]) return;
    const int mi = cta_mat[pair];
    const JMat mt = mats[mi];
    const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, t = lane & 3;
    if (!j_pair_rows(mt, pair - mt.cta_begin, round, rmap, s_rows, tid)) return;
    __syncthreads();
    const double *QT = QTbuf + (int64_t)pair * (NPL * JP * JP);
    double qa[NPL][2][4][4];
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int k8 = 0; k8 < 4; ++k8) {
                const double *ap = QT + pl * (JP * JP) + (i * 16 + g) * JP + k8 * 8 + t;
                qa[pl][i][k8][0] = ap[0];
                qa[pl][i][k8][1] = ap[8 * JP];
                qa[pl][i][k8][2] = ap[4];
                qa[pl][i][k8][3] = ap[8 * JP + 4];
            }
    if (which == 0)
        j_apply<CPLX>(bufs, qa, work + mt.y_off, work + mt.yi_off, mt.ldy, s_rows, tid, split, nsplit);
    else
        j_apply<CPLX>(bufs, qa, work + mt.w_off, work + mt.wi_off, mt.ldw, s_rows, tid, split, nsplit);
}

template <bool CPLX>
__global__ void __launch_bounds__(JTHREADS)
    jacobi_apply_kernel(double *__restrict__ work, const JMat *__restrict__ mats, const int *__restrict__ cta_mat,
                        const int *__restrict__ rmap, int round, const double *__restrict__ QTbuf,
                        const int *__restrict__ flags) {
    extern __shared__ __align__(16) double jsmem[];
    jacobi_apply_body<CPLX>(jsmem, work, mats, cta_mat, rmap, round, QTbuf, flags, blockIdx.x, gridDim.x, blockIdx.y,
                            blockIdx.z);
}

// Small-block regime: one launch per round.  For matrices of a few hundred columns the three phases of a pair are a few
// microseconds of streaming around the rotation chain of the pivot solver, and the launch boundaries between them cost as
// much as the streaming itself; here one CTA per pair runs them back to back (no column split; G, Q^T and the flag go
// through the same global buffers, ordered by the CTA barrier).
__global__ void __launch_bounds__(JTHREADS)
    jacobi_round_fused_kernel(double *work, const JMat *__restrict__ mats, const int *__restrict__ cta_mat,
                              const int *__restrict__ rmap, int round, const int *__restrict__ done, int *rot_count,
                              double tol_scale, double *Gbuf, double *QTbuf, int *flags, int inner_sweeps) {
    extern __shared__ __align__(16) double jsmem[];
    const int pair = blockIdx.x;
    jacobi_gram_body<false>(jsmem, work, mats, cta_mat, rmap, round, done, Gbuf, 0, 1, pair);
    __syncthreads();
    jacobi_eig_v3_body(mats, cta_mat, rot_count, done, tol_scale, Gbuf, 1, QTbuf, flags, inner_sweeps, round, pair);
    __syncthreads();
    jacobi_apply_body<false>(jsmem, work, mats, cta_mat, rmap, round, QTbuf, flags, 0, 1, pair, 0);
    __syncthreads();
    jacobi_apply_body<false>(jsmem, work, mats, cta_mat, rmap, round, QTbuf, flags, 0, 1, pair, 1);
}

// ---- init / finalize kernels ---------------------------------------------------------------------
// mats[b].amax = max |a_ij| over the m x n entries of A (and Ai); amax must be 0 on entry.  grid (chunks, nmat), 256
// threads.  Non-negative doubles order like their bit patterns, so the CTA maxima combine exactly by an integer atomicMax.
// The block scale pow2_scale(amax) (scaling.cuh) follows; every later norm and Gram entry is formed on scale * A
__global__ void __launch_bounds__(256) jacobi_amax_kernel(JMat *__restrict__ mats, const double *__restrict__ A,
                                                          const double *__restrict__ Ai) {
    __shared__ double red[32];
    JMat *mt = mats + blockIdx.y;
    const int64_t mn = (int64_t)mt->m * mt->n;
    const int64_t a0 = mt->a_off;
    double amax = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < mn; e += (int64_t)gridDim.x * blockDim.x) {
        amax = fmax(amax, fabs(A[a0 + e]));
        if (Ai) amax = fmax(amax, fabs(Ai[a0 + e]));
    }
    amax = warp_max(amax);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) amax = fmax(amax, red[w]);
        if (amax > 0.0)
            atomicMax(reinterpret_cast<unsigned long long *>(&mt->amax), (unsigned long long)__double_as_longlong(amax));
    }
}

static void launch_amax(const std::vector<JMat> &mats, JMat *d_mats, const double *A, const double *Ai, cudaStream_t st) {
    int64_t max_elems = 0;
    for (auto &mt : mats) max_elems = std::max<int64_t>(max_elems, (int64_t)mt.m * mt.n);
    const int64_t gx = std::min<int64_t>(std::max<int64_t>(1, (max_elems + 4095) / 4096), 1024);
    jacobi_amax_kernel<<<dim3((unsigned)gx, (unsigned)mats.size()), 256, 0, st>>>(d_mats, A, Ai);
}

// squared row norms (first m entries) and column norms (next n entries) of every scale * A: grid (m + n, nmat).
// Ai (complex input, else NULL): imaginary part, |a|^2 = re^2 + im^2
__global__ void __launch_bounds__(128) svd_prep_kernel(double *__restrict__ work, const JMat *__restrict__ mats,
                                                       const double *__restrict__ A, const double *__restrict__ Ai) {
    __shared__ double red[32];
    JMat mt = mats[blockIdx.y];
    const int v = blockIdx.x;
    if (v >= mt.m + mt.n) return;
    mt.scale = pow2_scale(mt.amax);   // (the host stores the same value in mats before svd_init_kernel)
    const double *a = A + mt.a_off;
    double s = 0.0;
    if (v < mt.m) {
        for (int c = threadIdx.x; c < mt.n; c += blockDim.x) {
            double x = a[(int64_t)v * mt.n + c] * mt.scale;
            s = fma(x, x, s);
            if (Ai) {
                x = Ai[mt.a_off + (int64_t)v * mt.n + c] * mt.scale;
                s = fma(x, x, s);
            }
        }
    } else {
        const int c = v - mt.m;
        for (int r = threadIdx.x; r < mt.m; r += blockDim.x) {
            double x = a[(int64_t)r * mt.n + c] * mt.scale;
            s = fma(x, x, s);
            if (Ai) {
                x = Ai[mt.a_off + (int64_t)r * mt.n + c] * mt.scale;
                s = fma(x, x, s);
            }
        }
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) work[mt.prep_off + v] = s;
}

// SVD init: Y[r] = vector perm[r] of scale * A (rows of A, or columns if transposed -- not conjugated), zero padded;
// W = permutation.  Ai (complex input, else NULL): imaginary part into Yi (Wi stays zero).  grid (chunks, nmat)
__global__ void __launch_bounds__(256) svd_init_kernel(double *__restrict__ work, const JMat *__restrict__ mats,
                                                       const int *__restrict__ perm, const double *__restrict__ A,
                                                       const double *__restrict__ Ai) {
    const JMat mt = mats[blockIdx.y];
    double *Y = work + mt.y_off;
    double *W = work + mt.w_off;
    const double *a = A + mt.a_off;
    const int *pm = perm + mt.perm_off;
    const int64_t ny = (int64_t)mt.q * mt.p;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < ny; e += stride) {
        int r = (int)(e / mt.p), c = (int)(e % mt.p);
        int src = pm[r];
        const int64_t ia = mt.transposed ? (int64_t)c * mt.n + src : (int64_t)src * mt.n + c;
        Y[(int64_t)r * mt.ldy + c] = a[ia] * mt.scale;
        if (Ai) work[mt.yi_off + (int64_t)r * mt.ldy + c] = Ai[mt.a_off + ia] * mt.scale;
    }
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < mt.qp; e += stride)
        W[e * mt.ldw + (e < mt.q ? pm[e] : e)] = 1.0;
}

// eigh init: Y = scale * A + shift*I.  scale[mat] and shift[mat] are set by eigh_shift_kernel (after jacobi_amax_kernel).
// CPLX: Ai is the imaginary plane of a Hermitian A; the norm is over both planes and amax (jacobi_amax_kernel) covers both
template <bool CPLX>
__global__ void __launch_bounds__(256) eigh_shift_kernel(JMat *__restrict__ mats, const double *__restrict__ A,
                                                         const double *__restrict__ Ai) {
    __shared__ double red[32];
    JMat *mt = mats + blockIdx.x;
    const double *a = A + mt->a_off;
    const double scale = pow2_scale(mt->amax);
    const int64_t nn = (int64_t)mt->n * mt->n;
    double s = 0.0;
    for (int64_t e = threadIdx.x; e < nn; e += blockDim.x) {
        const double x = a[e] * scale;
        s = fma(x, x, s);
        if constexpr (CPLX) {
            const double y = Ai[mt->a_off + e] * scale;
            s = fma(y, y, s);
        }
    }
    s = block_sum(s, red);
    // (no absolute term: the scaled block has max |a| in [1, 2), and a zero block needs no shift -- W = 0 exactly)
    if (threadIdx.x == 0) {
        mt->scale = scale;
        mt->shift = 1.0625 * sqrt(s);
    }
}

// CPLX: Y = scale * (A + A^H) / 2 + shift*I -- the real plane symmetrised, the imaginary plane (Yi) antisymmetrised
template <bool CPLX>
__global__ void __launch_bounds__(256) eigh_init_kernel(double *__restrict__ work, const JMat *__restrict__ mats,
                                                        const double *__restrict__ A, const double *__restrict__ Ai) {
    const JMat mt = mats[blockIdx.y];
    double *Y = work + mt.y_off;
    double *W = work + mt.w_off;
    const double *a = A + mt.a_off;
    const int64_t ny = (int64_t)mt.q * mt.p;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < ny; e += stride) {
        int r = (int)(e / mt.p), c = (int)(e % mt.p);
        // symmetrise (use both triangles) like a Hermitian solver would see one triangle
        double v = 0.5 * (a[(int64_t)r * mt.n + c] * mt.scale + a[(int64_t)c * mt.n + r] * mt.scale);
        if (r == c) v += mt.shift;
        Y[(int64_t)r * mt.ldy + c] = v;
        if constexpr (CPLX) {
            const double *ai = Ai + mt.a_off;
            work[mt.yi_off + (int64_t)r * mt.ldy + c] =
                0.5 * (ai[(int64_t)r * mt.n + c] * mt.scale - ai[(int64_t)c * mt.n + r] * mt.scale);
        }
    }
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < mt.qp; e += stride)
        W[e * mt.ldw + e] = 1.0;
}

// row norms of Y: grid (max_q, nmat), 128 threads.  A row whose sum of squares is below 2^-900 (squares may have
// underflowed: rows graded far below the block's largest entry) is summed again scaled by the power of two of its largest
// entry; every other row gets the plain sum, as it always did.
__global__ void __launch_bounds__(128) jacobi_norms_kernel(double *__restrict__ work, const JMat *__restrict__ mats) {
    __shared__ double red[32];
    __shared__ double s_bc;
    const JMat mt = mats[blockIdx.y];
    const int r = blockIdx.x;
    if (r >= mt.q) return;
    const double *y = work + mt.y_off + (int64_t)r * mt.ldy;
    const double *yi = work + mt.yi_off + (int64_t)r * mt.ldy;
    double s = 0.0;
    for (int c = threadIdx.x; c < mt.p; c += blockDim.x) s = fma(y[c], y[c], s);
    if (mt.cplx)
        for (int c = threadIdx.x; c < mt.p; c += blockDim.x) s = fma(yi[c], yi[c], s);
    s = block_sum(s, red);
    if (threadIdx.x == 0) s_bc = s;
    __syncthreads();
    s = s_bc;
    if (s >= 0x1p-900 || s != s) {
        if (threadIdx.x == 0) work[mt.snorm_off + r] = sqrt(s);
        return;
    }
    double mx = 0.0;
    for (int c = threadIdx.x; c < mt.p; c += blockDim.x) {
        mx = fmax(mx, fabs(y[c]));
        if (mt.cplx) mx = fmax(mx, fabs(yi[c]));
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, red[w]);
        s_bc = pow2_scale(mx);
    }
    __syncthreads();
    const double sc = s_bc;
    double t = 0.0;
    for (int c = threadIdx.x; c < mt.p; c += blockDim.x) {
        double x = y[c] * sc;
        t = fma(x, x, t);
        if (mt.cplx) {
            x = yi[c] * sc;
            t = fma(x, x, t);
        }
    }
    t = block_sum(t, red);
    if (threadIdx.x == 0) work[mt.snorm_off + r] = sqrt(t) / sc;
}

// After a sweep, on the device: active-set bookkeeping of every matrix that is still iterating (one CTA per matrix).
// Rows ordered by descending norm (ties by index: the order std::stable_sort gives), rows with norm <= defl behind the
// active ones and out of the iteration; row map, nb_act, n_act updated in place, (nb_act, n_act) also to `act_out` for the
// host's launch geometry.  q <= J_REORDER_MAX (bitonic sort in shared memory).
constexpr int J_REORDER_MAX = 4096;
__global__ void __launch_bounds__(1024) jacobi_reorder_kernel(const double *__restrict__ work, JMat *mats, int *rmap,
                                                             const int *__restrict__ done, const int *__restrict__ rot,
                                                             int *__restrict__ act_out) {
    extern __shared__ __align__(16) unsigned char rsm[];
    __shared__ int s_nact;
    const int mi = blockIdx.x, tid = threadIdx.x;
    JMat &mt = mats[mi];
    const int q = mt.q;
    if (done[mi] || rot[mi] == 0 || !(mt.defl > 0.0)) {
        if (tid == 0) {
            act_out[2 * mi] = mt.nb_act;
            act_out[2 * mi + 1] = mt.n_act;
        }
        return;
    }
    int np2 = 2;
    while (np2 < q) np2 <<= 1;
    double *key = reinterpret_cast<double *>(rsm);
    int *idx = reinterpret_cast<int *>(rsm + (size_t)np2 * sizeof(double));
    const double *nrm = work + mt.snorm_off;
    for (int i = tid; i < np2; i += blockDim.x) {
        key[i] = i < q ? nrm[i] : -1.0;       // padding sorts behind every real row (norms are >= 0)
        idx[i] = i;
    }
    if (tid == 0) s_nact = 0;
    __syncthreads();
    for (int k = 2; k <= np2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < np2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const double ki = key[i], kl = key[l];
                    const int ii = idx[i], il = idx[l];
                    const bool i_first = ki > kl || (ki == kl && ii < il);     // i belongs before l in the final order
                    const bool want_first = (i & k) == 0;
                    if (i_first != want_first) {
                        key[i] = kl;
                        key[l] = ki;
                        idx[i] = il;
                        idx[l] = ii;
                    }
                }
            }
            __syncthreads();
        }
    }
    const double defl = mt.defl;
    for (int i = tid; i < q; i += blockDim.x)
        if (key[i] > defl && (i + 1 == q || !(key[i + 1] > defl))) s_nact = i + 1;
    int *rm = rmap + mt.rmap_off;
    for (int i = tid; i < mt.qp; i += blockDim.x) rm[i] = i < q ? idx[i] : i;
    __syncthreads();
    if (tid == 0) {
        const int n_act = s_nact;
        const int nb_act = j_nb_act(n_act, mt.nb);
        mt.nb_act = nb_act;
        mt.n_act = n_act;
        act_out[2 * mi] = nb_act;
        act_out[2 * mi + 1] = n_act;
    }
}

// SVD finalize: grid (max_k, nmat).  W Y0 = Y with W orthogonal (unitary) and the rows of Y orthogonal:
//   not transposed (Y0 = A):    A = W^H Y        -> U[:, r] = conj(W[r, :]),  VT[r, :] = Y[r, :] / s_r
//   transposed (Y0 = A^T):      A = Y^T conj(W)  -> U[:, r] = Y[r, :] / s_r,  VT[r, :] = conj(W[r, :])
// Ui, VTi (complex matrices, else NULL): the imaginary parts, from Yi and Wi
__global__ void __launch_bounds__(128)
    svd_finalize_kernel(const double *__restrict__ work, const JMat *__restrict__ mats, const int *__restrict__ perm,
                        double *__restrict__ U, double *__restrict__ Ui, double *__restrict__ S, double *__restrict__ VT,
                        double *__restrict__ VTi) {
    const JMat mt = mats[blockIdx.y];
    const int r = blockIdx.x;
    const int k = mt.q;
    if (r >= k) return;
    const int src = perm[mt.perm_off + r];
    const double s = work[mt.snorm_off + src];
    const double inv = (s > mt.defl && s > 0.0) ? 1.0 / s : 0.0;   // negligible direction: filled by the caller
    const double *y = work + mt.y_off + (int64_t)src * mt.ldy, *yi = work + mt.yi_off + (int64_t)src * mt.ldy;
    const double *w = work + mt.w_off + (int64_t)src * mt.ldw, *wi = work + mt.wi_off + (int64_t)src * mt.ldw;
    if (threadIdx.x == 0) S[mt.s_off + r] = s / mt.scale;     // exact: scale is a power of two
    const int64_t u0 = mt.u_off + r, vt0 = mt.vt_off + (int64_t)r * mt.n;
    if (mt.transposed) {  // Y rows: length m -> U[:, r];  W rows: length n -> VT[r, :]
        for (int i = threadIdx.x; i < mt.m; i += blockDim.x) {
            U[u0 + (int64_t)i * k] = y[i] * inv;
            if (Ui) Ui[u0 + (int64_t)i * k] = yi[i] * inv;
        }
        for (int c = threadIdx.x; c < mt.n; c += blockDim.x) {
            VT[vt0 + c] = w[c];
            if (VTi) VTi[vt0 + c] = -wi[c];
        }
    } else {  // Y rows: length n -> VT[r, :];  W rows: length m -> U[:, r]
        for (int c = threadIdx.x; c < mt.n; c += blockDim.x) {
            VT[vt0 + c] = y[c] * inv;
            if (VTi) VTi[vt0 + c] = yi[c] * inv;
        }
        for (int i = threadIdx.x; i < mt.m; i += blockDim.x) {
            U[u0 + (int64_t)i * k] = w[i];
            if (Ui) Ui[u0 + (int64_t)i * k] = -wi[i];
        }
    }
}

// eigh finalize: eigenvalue r (ascending) = (norm[perm[r]] - shift) / scale; V[:, r] = W[perm[r], :]
// CPLX: W Y0 = Y with W unitary and the rows of Y orthogonal, so W Y0^2 W^H is diagonal and the eigenvectors of Y0 are the
// columns of W^H: V[:, r] = conj(W[perm[r], :]) (svd_finalize_kernel writes Ui = -wi for the same reason)
template <bool CPLX>
__global__ void __launch_bounds__(128)
    eigh_finalize_kernel(const double *__restrict__ work, const JMat *__restrict__ mats, const int *__restrict__ perm,
                         double *__restrict__ Wout, double *__restrict__ V, double *__restrict__ Vi) {
    const JMat mt = mats[blockIdx.y];
    const int r = blockIdx.x;
    const int n = mt.n;
    if (r >= n) return;
    const int src = perm[mt.perm_off + r];
    const double *w = work + mt.w_off + (int64_t)src * mt.ldw;
    if (threadIdx.x == 0) Wout[mt.s_off + r] = (work[mt.snorm_off + src] - mt.shift) / mt.scale;
    double *v = V + mt.vt_off;
    for (int i = threadIdx.x; i < n; i += blockDim.x) v[(int64_t)i * n + r] = w[i];
    if constexpr (CPLX) {
        const double *wi = work + mt.wi_off + (int64_t)src * mt.ldw;
        double *vi = Vi + mt.vt_off;
        for (int i = threadIdx.x; i < n; i += blockDim.x) vi[(int64_t)i * n + r] = -wi[i];
    }
}

// ---- host driver -----------------------------------------------------------------------------------
// pivot eigen-solver: 3 = jacobi_eig_kernel_v3 (registers + shuffles, default), 1 = jacobi_eig_kernel (shared memory).
// Inner sweeps: ONE inner sweep makes a round cheaper, but the numerically low-rank two-site wave functions of a converged
// DMRG then need more outer sweeps: the default is 2.
static int g_eig_variant = 3;
static int env_fused_max_ld() {                     // B200_SVD_FUSED_LD: largest row length of the single-launch rounds (0: off)
    const char *e = getenv("B200_SVD_FUSED_LD");
    if (e == nullptr || *e == 0) return 256;
    const int n = atoi(e);
    return n >= 0 ? n : 256;
}
static int g_fused_max_ld = env_fused_max_ld();
static int env_inner_sweeps() {                     // B200_SVD_INNER=0..16 overrides the default (A/B runs of whole sweeps)
    const char *e = getenv("B200_SVD_INNER");
    if (e == nullptr || *e == 0) return J_INNER_SWEEPS;
    const int n = atoi(e);
    return (n >= 0 && n <= 16) ? n : J_INNER_SWEEPS;
}
static int g_eig_inner_sweeps = env_inner_sweeps();   // inner sweeps of version 3 (0: cross mode; version 1: fixed J_INNER_SWEEPS)
struct JLayout {
    std::vector<JMat> mats;
    std::vector<int> cta_mat;
    int64_t f64_elems = 0;     // doubles in the work area
    int64_t perm_elems = 0, rmap_elems = 0;
    int64_t g_off = 0, qt_off = 0;   // f64 offsets of the per-pair Gram partials and Q^T matrices
    int64_t off_flags = 0;
    int max_q = 0, max_nb = 0;
    // byte offsets of the integer regions inside the work buffer
    int64_t off_mats = 0, off_cta = 0, off_rot = 0, off_done = 0, off_perm = 0, off_rmap = 0, off_act = 0, total_bytes = 0;
};

static inline int64_t rup(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// cplx: complex SVD -- Y and W get planar imaginary parts, the Gram partials and Q^T matrices of a pair are complex
static void make_layout(int64_t nblocks, const int64_t *m, const int64_t *n, bool eigh, JLayout &L, bool cplx = false) {
    const int64_t cw = cplx ? 2 : 1;
    L.mats.resize((size_t)nblocks);
    int64_t off = 0;
    int cta = 0;
    int64_t perm = 0, rmap = 0;
    for (int64_t i = 0; i < nblocks; ++i) {
        JMat &mt = L.mats[(size_t)i];
        memset(&mt, 0, sizeof(JMat));
        mt.m = (int32_t)m[i];
        mt.n = (int32_t)(eigh ? m[i] : n[i]);
        mt.transposed = (!eigh && mt.m >= mt.n) ? 1 : 0;
        mt.q = std::min(mt.m, mt.n);
        mt.p = std::max(mt.m, mt.n);
        int nb = (int)((mt.q + JB - 1) / JB);
        if (nb < 2) nb = 2;
        if (nb & 1) ++nb;
        mt.nb = nb;
        mt.qp = nb * JB;
        mt.ldy = (int32_t)rup(mt.p, 16);
        mt.ldw = (int32_t)rup(mt.qp, 16);
        mt.y_off = off;
        off += (int64_t)mt.qp * mt.ldy;
        mt.w_off = off;
        off += (int64_t)mt.qp * mt.ldw;
        if (cplx) {
            mt.cplx = 1;
            mt.yi_off = off;
            off += (int64_t)mt.qp * mt.ldy;
            mt.wi_off = off;
            off += (int64_t)mt.qp * mt.ldw;
        }
        mt.snorm_off = off;
        off += rup(mt.qp, 16);
        mt.prep_off = off;
        off += rup((int64_t)mt.m + mt.n, 16);
        mt.cta_begin = cta;
        for (int c = 0; c < nb / 2; ++c) L.cta_mat.push_back((int)i);
        cta += nb / 2;
        mt.perm_off = (int32_t)perm;
        perm += mt.q;
        mt.rmap_off = (int32_t)rmap;
        rmap += mt.qp;
        mt.nb_act = nb;
        mt.n_act = mt.q;
        mt.defl = 0.0;
        mt.scale = 1.0;
        L.max_q = std::max(L.max_q, (int)mt.q);
        L.max_nb = std::max(L.max_nb, nb);
    }
    L.g_off = off;
    off += (int64_t)L.cta_mat.size() * J_NSPLIT_MAX * JP * JP * cw;
    L.qt_off = off;
    off += (int64_t)L.cta_mat.size() * JP * JP * cw;
    L.f64_elems = off;
    L.perm_elems = perm;
    L.rmap_elems = rmap;
    int64_t b = rup(off * (int64_t)sizeof(double), 256);
    L.off_mats = b;
    b += rup((int64_t)nblocks * (int64_t)sizeof(JMat), 256);
    L.off_cta = b;
    b += rup((int64_t)L.cta_mat.size() * 4, 256);
    L.off_rot = b;
    b += rup(nblocks * 4, 256);
    L.off_done = b;
    b += rup(nblocks * 4, 256);
    L.off_perm = b;
    b += rup(perm * 4 + 4, 256);
    L.off_rmap = b;
    b += rup(rmap * 4 + 4, 256);
    L.off_flags = b;
    b += rup((int64_t)L.cta_mat.size() * 4 + 4, 256);
    L.off_act = b;                     // (nb_act, n_act) per matrix, written by jacobi_reorder_kernel
    b += rup(nblocks * 8, 256);
    L.total_bytes = b;
}

// Host driver of the Jacobi iteration.  After every sweep the row norms are read back (q doubles per
// matrix): rows whose norm fell below the deflation threshold `defl` are numerically zero singular
// directions -- they are moved (logically, through the row map) behind the active rows and never touched
// again, so a numerically rank-deficient block only iterates on its significant rows.  Active rows are kept
// ordered by descending norm (de Rijk).
// cplx: the matrices are complex (layout made with cplx = true); the rounds run the complex instantiations of the kernels
static int run_jacobi(JLayout &L, char *work, cudaStream_t st, int32_t *info, int max_sweeps, bool cplx = false) {
    const int nmat = (int)L.mats.size();
    double *wf = reinterpret_cast<double *>(work);
    JMat *d_mats = reinterpret_cast<JMat *>(work + L.off_mats);
    int *d_cta = reinterpret_cast<int *>(work + L.off_cta);
    int *d_rot = reinterpret_cast<int *>(work + L.off_rot);
    int *d_done = reinterpret_cast<int *>(work + L.off_done);
    int *d_rmap = reinterpret_cast<int *>(work + L.off_rmap);
    double *d_G = wf + L.g_off;
    double *d_QT = wf + L.qt_off;
    int *d_flags = reinterpret_cast<int *>(work + L.off_flags);
    static bool attr_set = false;
    if (!attr_set) {
        for (const void *k : {(const void *)jacobi_gram_kernel<false>, (const void *)jacobi_apply_kernel<false>,
                              (const void *)jacobi_round_fused_kernel})
            B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, jacobi_smem_bytes<false>()));
        for (const void *k : {(const void *)jacobi_gram_kernel<true>, (const void *)jacobi_apply_kernel<true>})
            B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, jacobi_smem_bytes<true>()));
        // (q = 4096: 48 KB of keys and indices + the kernel's static shared memory is above the default limit)
        B200_CUDA_CHECK(cudaFuncSetAttribute(jacobi_reorder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             J_REORDER_MAX * 12));
        attr_set = true;
    }
    std::vector<int> rot((size_t)nmat), done((size_t)nmat, 0);
    std::vector<int> rmap((size_t)L.rmap_elems + 1, 0);
    for (int i = 0; i < nmat; ++i) {
        info[i] = -1;
        const JMat &mt = L.mats[(size_t)i];
        std::iota(rmap.begin() + mt.rmap_off, rmap.begin() + mt.rmap_off + mt.qp, 0);
    }
    B200_CUDA_CHECK(cudaMemcpyAsync(d_rmap, rmap.data(), rmap.size() * 4, cudaMemcpyHostToDevice, st));
    const int n_cta = (int)L.cta_mat.size();
    const double tol_scale = 2.0e-15;   // tol = tol_scale * sqrt(p): a few times the rounding noise of a length-p dot product
    const bool debug = getenv("B200_JACOBI_DEBUG") != nullptr;
    B200_CUDA_CHECK(cudaMemsetAsync(d_done, 0, (size_t)nmat * 4, st));
    int ndone = 0;
    int round_counter = 0;
    // active-set bookkeeping between the sweeps on the device (jacobi_reorder_kernel) unless a matrix is too large for its
    // shared-memory sort or B200_SVD_HOST_REORDER is set (A/B): then row norms come back to the host, one copy per matrix
    const bool dev_reorder = L.max_q <= J_REORDER_MAX && getenv("B200_SVD_HOST_REORDER") == nullptr;
    int *d_act = reinterpret_cast<int *>(work + L.off_act);
    std::vector<int> act((size_t)2 * nmat, 0);
    std::vector<double> nrm;
    std::vector<int> order;
    // one round in three launches, the streaming phases over nsplit column splits: Gram partials, pivot solver, P <- Q^T P
    // for Y and W.  Complex blocks always take it, with pivot solver 1
    auto split_round = [&](auto cplx_tag, int nsplit) -> int {
        constexpr bool CPLX = decltype(cplx_tag)::value;
        jacobi_gram_kernel<CPLX><<<dim3((unsigned)nsplit, (unsigned)n_cta), JTHREADS, jacobi_smem_bytes<CPLX>(), st>>>(
            wf, d_mats, d_cta, d_rmap, round_counter, d_done, d_G);
        B200_CHECK_LAUNCH();
        if (!CPLX && g_eig_variant == 3)
            jacobi_eig_kernel_v3<<<n_cta, JTHREADS, 0, st>>>(d_mats, d_cta, d_rot, d_done, tol_scale, d_G, nsplit, d_QT,
                                                           d_flags, g_eig_inner_sweeps, round_counter);
        else
            jacobi_eig_kernel<CPLX><<<n_cta, JTHREADS, 0, st>>>(d_mats, d_cta, d_rot, d_done, tol_scale, d_G, nsplit, d_QT,
                                                                d_flags, CPLX ? std::max(1, g_eig_inner_sweeps) : J_INNER_SWEEPS);
        B200_CHECK_LAUNCH();
        jacobi_apply_kernel<CPLX><<<dim3((unsigned)nsplit, (unsigned)n_cta, 2), JTHREADS, jacobi_smem_bytes<CPLX>(), st>>>(
            wf, d_mats, d_cta, d_rmap, round_counter, d_QT, d_flags);
        B200_CHECK_LAUNCH();
        return B200_OK;
    };
    for (int sweep = 0; sweep < max_sweeps && ndone < nmat; ++sweep) {
        int rounds = 1;
        for (int i = 0; i < nmat; ++i)
            if (!done[i]) rounds = std::max(rounds, L.mats[(size_t)i].nb_act - 1);
        B200_CUDA_CHECK(cudaMemsetAsync(d_rot, 0, (size_t)nmat * 4, st));
        // column splits: enough CTAs to fill the GPU ~3x with the pairs that are still active
        int act_pairs = 0, max_ld = 0;
        for (int i = 0; i < nmat; ++i)
            if (!done[i]) {
                act_pairs += L.mats[(size_t)i].nb_act / 2;
                max_ld = std::max(max_ld, std::max(L.mats[(size_t)i].ldy, L.mats[(size_t)i].ldw));
            }
        int nsplit = (3 * sm_count() + act_pairs - 1) / std::max(1, act_pairs);
        nsplit = std::max(1, std::min(nsplit, std::min(J_NSPLIT_MAX, (max_ld + JKC - 1) / JKC)));
        // small-block regime: all phases of a round in one launch (one CTA per pair, no column split)
        const bool fused = !cplx && g_eig_variant == 3 && max_ld <= g_fused_max_ld;
        for (int r = 0; r < rounds; ++r) {
            if (fused) {
                jacobi_round_fused_kernel<<<n_cta, JTHREADS, jacobi_smem_bytes<false>(), st>>>(
                    wf, d_mats, d_cta, d_rmap, round_counter, d_done, d_rot, tol_scale, d_G, d_QT, d_flags, g_eig_inner_sweeps);
                B200_CHECK_LAUNCH();
            } else {
                const int rc = cplx ? split_round(std::true_type(), nsplit) : split_round(std::false_type(), nsplit);
                if (rc) return rc;
            }
            ++round_counter;
        }
        jacobi_norms_kernel<<<dim3((unsigned)std::max(1, L.max_q), (unsigned)nmat), 128, 0, st>>>(wf, d_mats);
        B200_CHECK_LAUNCH();
        auto now_ms = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
        if (dev_reorder) {
            int np2 = 2;
            while (np2 < L.max_q) np2 <<= 1;
            jacobi_reorder_kernel<<<nmat, std::max(64, std::min(1024, np2 / 2)), (size_t)np2 * 12, st>>>(wf, d_mats, d_rmap, d_done, d_rot, d_act);
            B200_CHECK_LAUNCH();
            B200_CUDA_CHECK(cudaMemcpyAsync(act.data(), d_act, (size_t)nmat * 8, cudaMemcpyDeviceToHost, st));
        }
        const double t_issued = debug ? now_ms() : 0.0;
        B200_CUDA_CHECK(cudaMemcpyAsync(rot.data(), d_rot, (size_t)nmat * 4, cudaMemcpyDeviceToHost, st));
        B200_CUDA_CHECK(cudaStreamSynchronize(st));
        const double t_synced = debug ? now_ms() : 0.0;
        bool changed = false, mats_changed = false, remap = false;
        long tot = 0;
        for (int i = 0; i < nmat; ++i) {
            tot += rot[i];
            if (done[i]) continue;
            JMat &mt = L.mats[(size_t)i];
            if (rot[i] == 0) {
                done[i] = 1;
                info[i] = sweep + 1;
                ++ndone;
                changed = true;
                continue;
            }
            if (mt.defl <= 0.0) continue;
            if (dev_reorder) {        // the device has re-ordered the rows and updated its descriptors: mirror the geometry
                mt.nb_act = act[(size_t)2 * i];
                mt.n_act = act[(size_t)2 * i + 1];
                continue;
            }
            // re-order the logical rows: active rows by descending norm, then the deflated ones
            nrm.resize((size_t)mt.q);
            B200_CUDA_CHECK(cudaMemcpy(nrm.data(), wf + mt.snorm_off, (size_t)mt.q * sizeof(double), cudaMemcpyDeviceToHost));
            order.resize((size_t)mt.q);
            std::iota(order.begin(), order.end(), 0);
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return nrm[a] > nrm[b]; });
            int n_act = 0;
            while (n_act < mt.q && nrm[order[n_act]] > mt.defl) ++n_act;
            const int nb_act = j_nb_act(n_act, mt.nb);
            int *rm = rmap.data() + mt.rmap_off;
            // physical padding rows (>= q) stay at the very end of the logical order
            for (int k = 0; k < mt.q; ++k) rm[k] = order[k];
            for (int k = mt.q; k < mt.qp; ++k) rm[k] = k;
            if (nb_act != mt.nb_act || n_act != mt.n_act) {
                mt.nb_act = nb_act;
                mt.n_act = n_act;
                mats_changed = true;
            }
            remap = true;
        }
        if (ndone < nmat) {
            if (changed)
                B200_CUDA_CHECK(cudaMemcpyAsync(d_done, done.data(), (size_t)nmat * 4, cudaMemcpyHostToDevice, st));
            if (mats_changed)   // (never for eigh: its device-side `shift` must not be overwritten)
                B200_CUDA_CHECK(cudaMemcpyAsync(d_mats, L.mats.data(), (size_t)nmat * sizeof(JMat), cudaMemcpyHostToDevice, st));
            if (remap)
                B200_CUDA_CHECK(cudaMemcpyAsync(d_rmap, rmap.data(), rmap.size() * 4, cudaMemcpyHostToDevice, st));
            // no synchronisation: the sources are pageable, i.e. staged by the driver before cudaMemcpyAsync returns, and
            // the next sweep's kernels are ordered behind the copies on the stream
        }
        if (debug)   // host waited `wait` ms for the sweep's kernels; during `host gap` the GPU has nothing to do
            fprintf(stderr, "[jacobi] sweep %d: %ld rotated pairs, %d rounds (%s), %d/%d matrices done, n_act[0]=%d/%d, wait %.3f ms, "
                    "host gap %.3f ms\n", sweep, tot, rounds, fused ? "fused" : "split", ndone, nmat, L.mats[0].n_act, L.mats[0].q,
                    t_synced - t_issued, now_ms() - t_synced);
    }
    (void)d_cta;
    return B200_OK;
}

// sort (descending by norm) on the host; returns permutation pool
static int sort_norms(JLayout &L, char *work, cudaStream_t st, bool ascending, std::vector<int> &perm) {
    const int nmat = (int)L.mats.size();
    double *wf = reinterpret_cast<double *>(work);
    JMat *d_mats = reinterpret_cast<JMat *>(work + L.off_mats);
    dim3 grid((unsigned)std::max(1, L.max_q), (unsigned)nmat);
    jacobi_norms_kernel<<<grid, 128, 0, st>>>(wf, d_mats);
    B200_CHECK_LAUNCH();
    perm.assign((size_t)L.perm_elems + 1, 0);
    std::vector<double> nrm;
    for (int i = 0; i < nmat; ++i) {
        JMat &mt = L.mats[(size_t)i];
        nrm.resize((size_t)mt.q);
        B200_CUDA_CHECK(cudaMemcpyAsync(nrm.data(), wf + mt.snorm_off, (size_t)mt.q * sizeof(double),
                                        cudaMemcpyDeviceToHost, st));
        B200_CUDA_CHECK(cudaStreamSynchronize(st));
        if (mt.defl > 0.0) {   // number of significant (non-negligible) directions
            int na = 0;
            for (int k = 0; k < mt.q; ++k) na += (nrm[k] > mt.defl) ? 1 : 0;
            mt.n_act = na;
        }
        int *pp = perm.data() + mt.perm_off;
        std::iota(pp, pp + mt.q, 0);
        if (ascending)
            std::stable_sort(pp, pp + mt.q, [&](int a, int b) { return nrm[a] < nrm[b]; });
        else
            std::stable_sort(pp, pp + mt.q, [&](int a, int b) { return nrm[a] > nrm[b]; });
    }
    int *d_perm = reinterpret_cast<int *>(work + L.off_perm);
    B200_CUDA_CHECK(cudaMemcpyAsync(d_perm, perm.data(), perm.size() * 4, cudaMemcpyHostToDevice, st));
    return B200_OK;
}

}  // namespace b200

using namespace b200;

static int g_svd_deflation = 1;
static double g_svd_defl_rel = 0.0;   // additional relative deflation threshold (0: only the rounding-level one)
extern "C" double b200_svd_set_deflation_tol(double tol_rel) {
    double old = g_svd_defl_rel;
    g_svd_defl_rel = tol_rel > 0.0 ? tol_rel : 0.0;
    return old;
}
extern "C" int b200_svd_set_eig_variant(int variant) {
    int old = g_eig_variant;
    if (variant == 1 || variant == 3) g_eig_variant = variant;
    return old;
}

extern "C" int b200_svd_set_eig_inner_sweeps(int n) {
    int old = g_eig_inner_sweeps;
    if (n >= 0 && n <= 16) g_eig_inner_sweeps = n;   // 0: cross mode of version 3 (see jacobi_eig_kernel_v3)
    return old;
}

extern "C" int b200_svd_set_fused_max_ld(int max_ld) {
    int old = g_fused_max_ld;
    if (max_ld >= 0) g_fused_max_ld = max_ld;
    return old;
}

extern "C" int b200_svd_set_deflation(int on) {
    int old = g_svd_deflation;
    g_svd_deflation = on ? 1 : 0;
    return old;
}

extern "C" int64_t b200_block_svd_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    if (nblocks <= 0) return 256;
    JLayout L;
    make_layout(nblocks, m, n, false, L);
    return L.total_bytes;
}

// real (Ai == NULL) and complex (planar: A + i Ai -> U + i Ui, VT + i VTi) block SVD: one host driver
static int block_svd_impl(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off, const int64_t *u_off,
                          const int64_t *s_off, const int64_t *vt_off, const double *A, const double *Ai, double *U,
                          double *Ui, double *S, double *VT, double *VTi, void *work_dev, int64_t work_bytes, int32_t *info,
                          int32_t *nact_host, int32_t *transposed_host, b200_stream_t stream) {
    if (nblocks <= 0) return B200_OK;
    if (nblocks > 65535) return set_error(B200_ERR_ARG, "too many blocks for one SVD batch");
    const bool cplx = Ai != nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    const double t_start = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    JLayout L;
    make_layout(nblocks, m, n, false, L, cplx);
    if (work_bytes < L.total_bytes) return set_error(B200_ERR_ARG, "SVD work buffer too small: %lld < %lld",
                                                     (long long)work_bytes, (long long)L.total_bytes);
    for (int64_t i = 0; i < nblocks; ++i) {
        if (m[i] <= 0 || n[i] <= 0) return set_error(B200_ERR_ARG, "empty block in SVD batch");
        JMat &mt = L.mats[(size_t)i];
        mt.a_off = a_off[i];
        mt.u_off = u_off[i];
        mt.s_off = s_off[i];
        mt.vt_off = vt_off[i];
    }
    char *work = reinterpret_cast<char *>(work_dev);
    const int nmat = (int)nblocks;
    B200_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)L.off_mats, st));
    B200_CUDA_CHECK(cudaMemcpyAsync(work + L.off_mats, L.mats.data(), (size_t)nmat * sizeof(JMat),
                                    cudaMemcpyHostToDevice, st));
    B200_CUDA_CHECK(cudaMemcpyAsync(work + L.off_cta, L.cta_mat.data(), L.cta_mat.size() * 4, cudaMemcpyHostToDevice, st));
    JMat *d_mats = reinterpret_cast<JMat *>(work + L.off_mats);
    double *wf = reinterpret_cast<double *>(work);
    {
        // orientation + pre-sort: orthogonalise the side whose Gram matrix is closer to diagonal (for square
        // blocks), vectors ordered by descending norm (de Rijk); both from one pass over A.
        // Both, and the whole iteration, work on scale * A (jacobi_amax_kernel), so that no sum of squares over- or
        // underflows for any finite block; the threshold `defl` is in the same units.
        int max_mn = 0;
        for (auto &mt : L.mats) max_mn = std::max(max_mn, mt.m + mt.n);
        launch_amax(L.mats, d_mats, A, Ai, st);
        B200_CHECK_LAUNCH();
        svd_prep_kernel<<<dim3((unsigned)max_mn, (unsigned)nmat), 128, 0, st>>>(wf, d_mats, A, Ai);
        B200_CHECK_LAUNCH();
        B200_CUDA_CHECK(cudaMemcpyAsync(L.mats.data(), d_mats, (size_t)nmat * sizeof(JMat), cudaMemcpyDeviceToHost, st));
        B200_CUDA_CHECK(cudaStreamSynchronize(st));   // L.mats (amax) is read below
        std::vector<int> perm0((size_t)L.perm_elems + 1, 0);
        std::vector<double> nr;
        bool changed = false;
        for (int i = 0; i < nmat; ++i) {
            JMat &mt = L.mats[(size_t)i];
            mt.scale = pow2_scale(mt.amax);
            nr.resize((size_t)mt.m + mt.n);
            B200_CUDA_CHECK(cudaMemcpyAsync(nr.data(), wf + mt.prep_off, nr.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
            B200_CUDA_CHECK(cudaStreamSynchronize(st));
            double fro2 = 0.0;
            {
                for (int r = 0; r < mt.m; ++r) fro2 += nr[r];
                mt.defl = g_svd_deflation ? std::max(16.0 * 2.220446049250313e-16 * sqrt((double)mt.p), g_svd_defl_rel) * sqrt(fro2) : 0.0;
                // an all-zero block: every direction is negligible (norm 0 <= 0), so it is fully deflated (n_act = 0) and
                // the caller completes both sides; the smallest positive threshold keeps the `defl > 0` bookkeeping on
                if (g_svd_deflation && fro2 == 0.0) mt.defl = std::numeric_limits<double>::min();
                changed = true;
            }
            if (mt.m == mt.n) {
                double r4 = 0.0, c4 = 0.0;
                for (int r = 0; r < mt.m; ++r) r4 += nr[r] * nr[r];
                for (int c = 0; c < mt.n; ++c) c4 += nr[mt.m + c] * nr[mt.m + c];
                int tr = (c4 > r4) ? 1 : 0;
                if (tr != mt.transposed) {
                    mt.transposed = tr;
                    changed = true;
                }
            }
            const double *vn = mt.transposed ? nr.data() + mt.m : nr.data();
            int *pp = perm0.data() + mt.perm_off;
            std::iota(pp, pp + mt.q, 0);
            std::stable_sort(pp, pp + mt.q, [&](int a, int b) { return vn[a] > vn[b]; });
            // vn = SQUARED norms: vectors that are negligible from the start never enter the active set
            // (Y is filled in this order, so the active rows are the first n_act logical = physical rows)
            if (mt.defl > 0.0) {
                int n_act = 0;
                while (n_act < mt.q && vn[pp[n_act]] > mt.defl * mt.defl) ++n_act;
                mt.n_act = n_act;
                mt.nb_act = j_nb_act(n_act, mt.nb);
                changed = true;
            }
        }
        if (changed)
            B200_CUDA_CHECK(cudaMemcpyAsync(work + L.off_mats, L.mats.data(), (size_t)nmat * sizeof(JMat),
                                            cudaMemcpyHostToDevice, st));
        int *d_perm = reinterpret_cast<int *>(work + L.off_perm);
        B200_CUDA_CHECK(cudaMemcpyAsync(d_perm, perm0.data(), perm0.size() * 4, cudaMemcpyHostToDevice, st));
        int64_t max_elems = 0;
        for (auto &mt : L.mats) max_elems = std::max<int64_t>(max_elems, (int64_t)mt.q * mt.p);
        int64_t gx = std::min<int64_t>(std::max<int64_t>(1, (max_elems + 1023) / 1024), 2048);
        svd_init_kernel<<<dim3((unsigned)gx, (unsigned)nmat), 256, 0, st>>>(wf, d_mats, d_perm, A, Ai);
        B200_CHECK_LAUNCH();
        B200_CUDA_CHECK(cudaStreamSynchronize(st));  // perm0 (host) must outlive the copy
    }
    const bool dbg = getenv("B200_JACOBI_DEBUG") != nullptr;
    auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_prep = now();
    int rc = run_jacobi(L, work, st, info, 60, cplx);
    if (rc) return rc;
    const double t_jac = now();
    std::vector<int> perm;
    rc = sort_norms(L, work, st, false, perm);
    if (rc) return rc;
    svd_finalize_kernel<<<dim3((unsigned)std::max(1, L.max_q), (unsigned)nmat), 128, 0, st>>>(
        wf, d_mats, reinterpret_cast<int *>(work + L.off_perm), U, Ui, S, VT, VTi);
    B200_CHECK_LAUNCH();
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
    if (dbg)
        fprintf(stderr, "[svd] prep+init %.2f ms, jacobi %.2f ms (%d sweeps), sort+finalize %.2f ms, n_act %d/%d\n",
                t_prep - t_start, t_jac - t_prep, info[0], now() - t_jac, L.mats[0].n_act, L.mats[0].q);
    for (int i = 0; i < nmat; ++i) {
        if (nact_host) nact_host[i] = L.mats[(size_t)i].n_act;
        if (transposed_host) transposed_host[i] = L.mats[(size_t)i].transposed;
    }
    for (int i = 0; i < nmat; ++i)
        if (info[i] < 0) return set_error(B200_ERR_NOCONV, "block Jacobi SVD did not converge for block %d", i);
    return B200_OK;
}

extern "C" int b200_block_svd_f64(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                                  const int64_t *u_off, const int64_t *s_off, const int64_t *vt_off, const double *A,
                                  double *U, double *S, double *VT, void *work_dev, int64_t work_bytes,
                                  int32_t *info, int32_t *nact_host, int32_t *transposed_host, b200_stream_t stream) {
    return block_svd_impl(nblocks, m, n, a_off, u_off, s_off, vt_off, A, nullptr, U, nullptr, S, VT, nullptr, work_dev,
                          work_bytes, info, nact_host, transposed_host, stream);
}

extern "C" int64_t b200_block_svd_z_worksize(int64_t nblocks, const int64_t *m, const int64_t *n) {
    if (nblocks <= 0) return 256;
    JLayout L;
    make_layout(nblocks, m, n, false, L, true);
    return L.total_bytes;
}

extern "C" int b200_block_svd_z(int64_t nblocks, const int64_t *m, const int64_t *n, const int64_t *a_off,
                                const int64_t *u_off, const int64_t *s_off, const int64_t *vt_off, const double *A_re,
                                const double *A_im, double *U_re, double *U_im, double *S, double *VT_re, double *VT_im,
                                void *work_dev, int64_t work_bytes, int32_t *info, int32_t *nact_host,
                                int32_t *transposed_host, b200_stream_t stream) {
    if (nblocks > 0 && (A_re == nullptr || A_im == nullptr))
        return set_error(B200_ERR_ARG, "complex SVD: both planes of A are needed");
    return block_svd_impl(nblocks, m, n, a_off, u_off, s_off, vt_off, A_re, A_im, U_re, U_im, S, VT_re, VT_im, work_dev,
                          work_bytes, info, nact_host, transposed_host, stream);
}

extern "C" int64_t b200_block_eigh_worksize(int64_t nblocks, const int64_t *n) {
    if (nblocks <= 0) return 256;
    JLayout L;
    make_layout(nblocks, n, n, true, L);
    return L.total_bytes;
}

// real (Ai == NULL) and complex Hermitian (planar: A + i Ai -> V + i Vi, W real) block eigh: one host driver
static int block_eigh_impl(int64_t nblocks, const int64_t *n, const int64_t *a_off, const int64_t *w_off,
                           const int64_t *v_off, const double *A, const double *Ai, double *Wout, double *V, double *Vi,
                           void *work_dev, int64_t work_bytes, int32_t *info, b200_stream_t stream) {
    if (nblocks <= 0) return B200_OK;
    if (nblocks > 65535) return set_error(B200_ERR_ARG, "too many blocks for one eigh batch");
    const bool cplx = Ai != nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    JLayout L;
    make_layout(nblocks, n, n, true, L, cplx);
    if (work_bytes < L.total_bytes) return set_error(B200_ERR_ARG, "eigh work buffer too small");
    for (int64_t i = 0; i < nblocks; ++i) {
        if (n[i] <= 0) return set_error(B200_ERR_ARG, "empty block in eigh batch");
        JMat &mt = L.mats[(size_t)i];
        mt.a_off = a_off[i];
        mt.s_off = w_off[i];
        mt.vt_off = v_off[i];
    }
    char *work = reinterpret_cast<char *>(work_dev);
    const int nmat = (int)nblocks;
    B200_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)L.off_mats, st));
    B200_CUDA_CHECK(cudaMemcpyAsync(work + L.off_mats, L.mats.data(), (size_t)nmat * sizeof(JMat),
                                    cudaMemcpyHostToDevice, st));
    B200_CUDA_CHECK(cudaMemcpyAsync(work + L.off_cta, L.cta_mat.data(), L.cta_mat.size() * 4, cudaMemcpyHostToDevice, st));
    JMat *d_mats = reinterpret_cast<JMat *>(work + L.off_mats);
    double *wf = reinterpret_cast<double *>(work);
    launch_amax(L.mats, d_mats, A, Ai, st);
    B200_CHECK_LAUNCH();
    if (cplx)
        eigh_shift_kernel<true><<<nmat, 256, 0, st>>>(d_mats, A, Ai);
    else
        eigh_shift_kernel<false><<<nmat, 256, 0, st>>>(d_mats, A, nullptr);
    B200_CHECK_LAUNCH();
    {
        int64_t max_elems = 0;
        for (auto &mt : L.mats) max_elems = std::max<int64_t>(max_elems, (int64_t)mt.q * mt.p);
        int64_t gx = std::min<int64_t>(std::max<int64_t>(1, (max_elems + 1023) / 1024), 2048);
        if (cplx)
            eigh_init_kernel<true><<<dim3((unsigned)gx, (unsigned)nmat), 256, 0, st>>>(wf, d_mats, A, Ai);
        else
            eigh_init_kernel<false><<<dim3((unsigned)gx, (unsigned)nmat), 256, 0, st>>>(wf, d_mats, A, nullptr);
        B200_CHECK_LAUNCH();
    }
    int rc = run_jacobi(L, work, st, info, 40, cplx);
    if (rc) return rc;
    std::vector<int> perm;
    rc = sort_norms(L, work, st, true, perm);
    if (rc) return rc;
    const dim3 fgrid((unsigned)std::max(1, L.max_q), (unsigned)nmat);
    int *d_perm = reinterpret_cast<int *>(work + L.off_perm);
    if (cplx)
        eigh_finalize_kernel<true><<<fgrid, 128, 0, st>>>(wf, d_mats, d_perm, Wout, V, Vi);
    else
        eigh_finalize_kernel<false><<<fgrid, 128, 0, st>>>(wf, d_mats, d_perm, Wout, V, nullptr);
    B200_CHECK_LAUNCH();
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int i = 0; i < nmat; ++i)
        if (info[i] < 0) return set_error(B200_ERR_NOCONV, "block Jacobi eigh did not converge for block %d", i);
    return B200_OK;
}

extern "C" int b200_block_eigh_f64(int64_t nblocks, const int64_t *n, const int64_t *a_off, const int64_t *w_off,
                                   const int64_t *v_off, const double *A, double *Wout, double *V, void *work_dev,
                                   int64_t work_bytes, int32_t *info, b200_stream_t stream) {
    return block_eigh_impl(nblocks, n, a_off, w_off, v_off, A, nullptr, Wout, V, nullptr, work_dev, work_bytes, info,
                           stream);
}

extern "C" int64_t b200_block_eigh_z_worksize(int64_t nblocks, const int64_t *n) {
    if (nblocks <= 0) return 256;
    JLayout L;
    make_layout(nblocks, n, n, true, L, true);
    return L.total_bytes;
}

extern "C" int b200_block_eigh_z(int64_t nblocks, const int64_t *n, const int64_t *a_off, const int64_t *w_off,
                                 const int64_t *v_off, const double *A_re, const double *A_im, double *W, double *V_re,
                                 double *V_im, void *work_dev, int64_t work_bytes, int32_t *info, b200_stream_t stream) {
    if (nblocks > 0 && (A_re == nullptr || A_im == nullptr || V_im == nullptr))
        return set_error(B200_ERR_ARG, "complex eigh: both planes of A and V are needed");
    return block_eigh_impl(nblocks, n, a_off, w_off, v_off, A_re, A_im, W, V_re, V_im, work_dev, work_bytes, info,
                           stream);
}
