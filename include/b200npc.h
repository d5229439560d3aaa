/* b200npc.h -- C ABI of libb200npc.so, the sm_90a device library behind tenpy_b200.
 *
 * This is the drop-in boundary for the two-site-DMRG hot path of tenpy/tenpy.  Each entry point
 * replaces one piece of the reference's native helper `tenpy/linalg/_npc_helper.pyx` (the only
 * compiled component of the reference) or one LAPACK/BLAS call site of `tenpy/linalg/np_conserved.py`;
 * the replaced reference code is cited next to each declaration as file:line (paths relative to the
 * reference checkout, "pyx" = tenpy/linalg/_npc_helper.pyx, "npc" = tenpy/linalg/np_conserved.py).
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success and a non-zero code on failure, with a
 *     human readable message available from b200_last_error() (thread local).
 *   - pointers named *_dev / A / B / C / X / Y point to DEVICE memory (HBM) of the current CUDA device;
 *     pointers named *_host (and all plan-construction inputs) point to HOST memory.
 *   - all floating point data is IEEE binary64 ("f64"); all indices/offsets are int64 counted in
 *     ELEMENTS (not bytes) relative to the base pointer of a packed block buffer.
 *   - a "packed block buffer" holds all stored blocks of one Array back to back, each block C-contiguous
 *     (row-major), block starts aligned to B200_BLOCK_ALIGN elements, padding zero-filled.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - no function falls back to the CPU: without a CUDA device they fail with B200_ERR_CUDA.
 */
#ifndef B200NPC_H
#define B200NPC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 1
#define B200_BLOCK_ALIGN 16 /* elements (=128 bytes) */

#define B200_OK 0
#define B200_ERR_ARG 1
#define B200_ERR_CUDA 2
#define B200_ERR_NOCONV 3
#define B200_ERR_ALLOC 4

typedef void *b200_stream_t;

/* ---- library / device ------------------------------------------------------------------------- */
int b200_abi_version(void);
const char *b200_last_error(void);
/* number of visible CUDA devices (0 if none / no driver) */
int b200_device_count(void);
/* properties of device `dev`: SM count, compute capability, total memory */
int b200_device_info(int dev, int *sm_count, int *cc_major, int *cc_minor, int64_t *mem_bytes);
/* number of kernels this library has launched since load (or since the last call with reset != 0) */
int64_t b200_kernel_launch_count(int reset);
/* self test of the FP64 tensor-core fragment layouts used by the kernels; out_host[0..3] receive the max
 * abs error of (m16n8k8 path, m8n8k4 path, grouped gemm 128-tile, grouped gemm 64-tile) on a fixed problem */
int b200_selftest(double *out_host);

/* ---- host-side integer bookkeeping (no device needed) ------------------------------------------- */
/* indices where consecutive rows of a row-major (n x width) int64 table differ, incl. 0 and n.
 * replaces charges._find_row_differences, charges.py:1922 / pyx:635.  out_host has room for n+1. */
int b200_find_row_differences(const int64_t *rows_host, int64_t n, int64_t width, int64_t *out_host,
                              int64_t *n_out);
/* argsort of the rows, LAST column is the primary key (np.lexsort(rows.T)); stable.
 * replaces the np.lexsort calls of pyx:1357-1377 (_tensordot_pre_sort) and npc:1441. */
int b200_lexsort_rows(const int64_t *rows_host, int64_t n, int64_t width, int64_t *perm_host);
/* charges modulo `mod` in place (mod==1: untouched). replaces ChargeInfo.make_valid charges.py:267/pyx:478 */
int b200_make_valid(int64_t *charges_host, int64_t n, int64_t qnumber, const int64_t *mod_host);
/* block index map: out[j] = i repeated blocksizes[i] times. replaces charges._map_blocks :1945/pyx:732 */
int b200_map_blocks(const int64_t *blocksizes_host, int64_t n, int64_t *out_host);

/* ---- tensordot: contraction plan + grouped GEMM --------------------------------------------------- */
/* A contraction plan is the host-precomputed charge-sector bookkeeping of one npc.tensordot
 * (replaces _tensordot_pre_sort pyx:1337, _tensordot_match_charges pyx:1382 and the packing loop
 * pyx:1710-1754 that fills CblasGemmBatch pyx:151).  Inputs describe the stored blocks of
 *   a: (n_a x rank_a) qindex table, contracted legs are the LAST n_contr columns, block i is a row-major
 *      (a_rows[i] x a_cols[i]) matrix at element offset a_off[i];
 *   b: (n_b x rank_b) qindex table, contracted legs are the FIRST n_contr columns, block j is a row-major
 *      (b_rows[j] x b_cols[j]) matrix at element offset b_off[j].
 * Output blocks C[r,c] = sum_k A[r,k] B[k,c] exist for every (row group r of a, column group c of b) with
 * at least one common contracted qindex tuple; they are lex-sorted like the reference (pyx:1772-1778). */
typedef struct b200_tdot_plan b200_tdot_plan;
int b200_tdot_plan_create(const int64_t *a_qdata_host, int64_t n_a, int32_t rank_a,
                          const int64_t *b_qdata_host, int64_t n_b, int32_t rank_b, int32_t n_contr,
                          const int64_t *a_rows_host, const int64_t *a_cols_host, const int64_t *a_off_host,
                          const int64_t *b_rows_host, const int64_t *b_cols_host, const int64_t *b_off_host,
                          b200_tdot_plan **plan_out);
/* sizes: number of C blocks, number of block products (GEMMs), C buffer size in elements, flops = sum 2mkn */
int b200_tdot_plan_info(const b200_tdot_plan *plan, int64_t *n_c, int64_t *n_pairs, int64_t *c_size,
                        double *flops);
/* fetch the result block table: c_qdata (n_c x (rank_a + rank_b - 2 n_contr)), offsets, rows, cols */
int b200_tdot_plan_get(const b200_tdot_plan *plan, int64_t *c_qdata_host, int64_t *c_off_host,
                       int64_t *c_rows_host, int64_t *c_cols_host);
/* fetch the block-product list (the list the reference hands to CblasGemmBatch, pyx:1743): for output block
 * t the products are p in [pair_ptr[t], pair_ptr[t+1]); pair_ptr has n_c+1 entries, the others n_pairs. */
int b200_tdot_plan_pairs(const b200_tdot_plan *plan, int64_t *pair_ptr_host, int64_t *a_off_host,
                         int64_t *b_off_host, int64_t *k_host);
/* execute: C = A . B for all blocks; C must hold c_size elements (padding is written as zero-free: the
 * caller zero-fills C once if it needs zero padding).  replaces CblasGemmBatch.run pyx:204-274. */
int b200_tdot_plan_run(b200_tdot_plan *plan, const double *A, const double *B, double *C,
                       b200_stream_t stream);
void b200_tdot_plan_destroy(b200_tdot_plan *plan);

/* Raw grouped GEMM without a plan object (used by the host-buffer plugin path and the benchmark):
 * n_tasks output blocks; task t is C_t (m[t] x n[t], row-major, at c_off[t]) = sum over pairs
 * p in [pair_ptr[t], pair_ptr[t+1]) of A_p (m[t] x k[p] at a_off[p]) . B_p (k[p] x n[t] at b_off[p]). */
int b200_grouped_gemm_f64(int64_t n_tasks, const int64_t *m_host, const int64_t *n_host,
                          const int64_t *c_off_host, const int64_t *pair_ptr_host, int64_t n_pairs,
                          const int64_t *k_host, const int64_t *a_off_host, const int64_t *b_off_host,
                          const double *A, const double *B, double *C, b200_stream_t stream);

/* ---- FP64 products on the int8 tensor path (wgmma s8 x s8, int32 accumulators in registers) --------------------- */
/* Ozaki splitting: each operand is cut into `slices` signed 7-bit digit planes (row-wise power-of-two scaling), the slice
 * products are exact int8 x int8 -> int32 tensor-core GEMMs fed by bulk async copies (TMA unit), the diagonals are summed
 * in FP64.  slices = 7: error ~1e-14 (|A||B|)_ij (Lanczos matvec), 8: FP64 rounding level.  Used by npc.tensordot for
 * large dense block products; replaces the dgemm of CblasGemmBatch.run pyx:204-274 there.
 * A split operand is an opaque device buffer of b200_ozaki_split_worksize(rows, k, slices) bytes holding a (rows x k)
 * matrix whose element (r, kk) is X[r*ld_row + kk*ld_k] (one of the two strides must be 1): pass (lda, 1) for the left
 * operand A (m x k, row-major) and (1, ldb) for the right operand B (k x n, row-major; rows = n).  Split operands can be
 * reused across products (the environments of a bond across all Lanczos iterations). */
int64_t b200_ozaki_split_worksize(int64_t rows, int64_t k, int32_t slices);
int b200_ozaki_split_f64(int64_t rows, int64_t k, const double *X, int64_t ld_row, int64_t ld_k, int32_t slices,
                         void *out_dev, int64_t out_bytes, b200_stream_t stream);
/* C (m x n, row-major, ldc) = (accumulate ? C : 0) + A . B from two split operands with the same k and slice count */
int b200_ozaki_mm_f64(int64_t m, int64_t n, int64_t k, int32_t slices, const void *a_split, const void *b_split,
                      double *C, int64_t ldc, int32_t accumulate, b200_stream_t stream);
/* split both operands into `work_dev` (b200_ozaki_gemm_worksize bytes) and multiply */
int64_t b200_ozaki_gemm_worksize(int64_t m, int64_t n, int64_t k, int32_t slices);
int b200_ozaki_gemm_f64(int64_t m, int64_t n, int64_t k, const double *A, int64_t lda, const double *B, int64_t ldb,
                        double *C, int64_t ldc, int32_t slices, int32_t accumulate, void *work_dev, int64_t work_bytes,
                        b200_stream_t stream);
/* every pipeline wait of the tensor-core kernel has a watchdog; returns B200_ERR_CUDA if one fired since the last call
 * (synchronises; for tests and debugging, never needed in a correct run) */
int b200_ozaki_check_abort(void);

/* ---- BLAS-1 on packed block buffers (Lanczos vector ops) ------------------------------------------ */
/* y += alpha x.  replaces Array.iadd_prefactor_other npc:2373 / pyx:860 (daxpy pyx:328-335) */
int b200_axpy_f64(int64_t n, double alpha, const double *X, double *Y, b200_stream_t stream);
/* x *= alpha.  replaces Array.iscale_prefactor npc:2386 / pyx:964 (dscal pyx:350-363) */
int b200_scal_f64(int64_t n, double alpha, double *X, b200_stream_t stream);
/* out_dev[0] = sum x_i y_i (deterministic two-stage reduction).  scratch_dev: >= B200_DOT_SCRATCH doubles.
 * replaces _inner_worker pyx:1791 (ddot pyx:1854-1871) and Array.norm npc:2241 (with X == Y). */
#define B200_DOT_SCRATCH 2048
int b200_dot_f64(int64_t n, const double *X, const double *Y, double *scratch_dev, double *out_dev,
                 b200_stream_t stream);
/* segment versions for Arrays with different block tables: seg_dev holds n_seg triples
 * (x_off, y_off, len) as int64 in device memory. */
int b200_axpy_segments_f64(int64_t n_seg, const int64_t *seg_dev, int64_t max_len, double alpha,
                           const double *X, double *Y, b200_stream_t stream);
int b200_dot_segments_f64(int64_t n_seg, const int64_t *seg_dev, int64_t max_len, const double *X,
                          const double *Y, double *scratch_dev, double *out_dev, b200_stream_t stream);
/* fused Lanczos step: w -= alpha*v1 + beta*v0 and out_dev[0] = |w|^2 in one pass (v0 may be NULL).
 * replaces the two iadd_prefactor_other + norm calls of krylov_based.py:665-671 */
int b200_lanczos_update_f64(int64_t n, double alpha, const double *V1, double beta, const double *V0,
                            double *W, double *scratch_dev, double *out_dev, b200_stream_t stream);
/* the same step with device-resident scalars: alpha = alpha_dev[0] (written there by b200_dot_f64),
 * beta = sqrt(beta2_dev[0]) (the |w|^2 of the previous step; beta2_dev / V0 may be NULL), and x *= 1/sqrt(norm2_dev[0]).
 * A Lanczos iteration (krylov_based.py:645-676) then needs no host round trip; the (alpha, beta) pairs are read back
 * in chunks for the tridiagonal eigenproblem and the convergence test.  Bit-identical to the host-scalar route.
 * Default; lanczos_params['device_scalars'] = False switches back. */
int b200_lanczos_update_dev_f64(int64_t n, const double *alpha_dev, const double *V1, const double *beta2_dev,
                                const double *V0, double *W, double *scratch_dev, double *out_dev,
                                b200_stream_t stream);
int b200_scal_rsqrt_dev_f64(int64_t n, const double *norm2_dev, double *X, b200_stream_t stream);
/* Krylov result assembly with complex coefficients (krylov_based.py:160 `_calc_result_full`, used for the Lanczos time
 * evolution): OUT = sum_{k < nvec} c_k v_k with c_k = coef_dev[2k] + i coef_dev[2k+1].  v_k is one plane of n doubles
 * (a real Krylov vector, in_planes = 1) or the planes [re; im] of 2n doubles (a packed complex one, in_planes = 2);
 * OUT is always the packed complex vector [re; im] of 2n doubles.  V_dev / coef_dev: the pointer table and the
 * coefficients in device memory; V_host: the same pointer table on the host, read for the argument checks only.  One
 * thread per element, FP64 accumulation in the order of the table.  Per complex output element it reads
 * 8 * in_planes * nvec bytes and writes 16 (the same result by axpy passes reads and rewrites OUT three times per vector).
 * Refused (B200_ERR_ARG, nothing launched): nvec outside 1..64, in_planes not 1 or 2, n < 0, a null pointer, OUT
 * overlapping a v_k.  n = 0 launches nothing. */
int b200_krylov_combine_f64(int64_t n, int64_t nvec, int64_t in_planes, const double *const *V_dev,
                            const double *const *V_host, const double *coef_dev, double *OUT, b200_stream_t stream);

/* ---- block data movement ------------------------------------------------------------------------- */
/* Strided N-d block copies: dst[doff + sum_i idx_i*dstride_i] = src[soff + sum_i idx_i*sstride_i].
 * task_dev holds n_tasks records of B200_COPY_REC int64: [soff, doff, n_elem, rank, shape[6], sstride[6],
 * dstride[6]] (iteration order = row-major over `shape`; make dstride the contiguous one for coalescing).
 * replaces _sliced_copy charges.py:1956/pyx:754, Array_itranspose pyx:813 (+ _imake_contiguous pyx:1000),
 * _combine_legs_worker pyx:1013, _split_legs_worker pyx:1136. */
#define B200_COPY_REC 22
#define B200_COPY_MAXRANK 6
int b200_copy_blocks_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                         const double *SRC, double *DST, b200_stream_t stream);
/* take along one axis: dst[o, j, i] = src[o, idx[j], i]; records of 7 int64:
 * [soff, doff, outer, n_keep, inner, src_len, idx_off]; idx_dev int64 index pool.
 * replaces Array.iproject npc:1914 (np.compress per block). */
#define B200_TAKE_REC 7
int b200_take_blocks_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                         const int64_t *idx_dev, const double *SRC, double *DST, b200_stream_t stream);
/* x[o, j, i] *= s[s_off + j]; records of 5 int64: [off, outer, len, inner, s_off].
 * replaces Array.iscale_axis npc:2108. */
#define B200_SCALE_REC 5
int b200_scale_axis_f64(int64_t n_tasks, const int64_t *task_dev, const int64_t *task_host,
                        const double *S_dev, double *X, b200_stream_t stream);

/* Batched Householder QR: block i is A_i (m_i x n_i, row-major at A + a_off[i]); Q_i (m_i x k_i, k = min(m, n)) is
 * written to Q + q_off[i], R_i (k_i x n_i, upper triangular, non-negative diagonal) to R + r_off[i].  One CTA per block,
 * one launch, no host round trip.  replaces the per-block np.linalg.qr of npc.qr (np_conserved.py:4139).  `work` =
 * device scratch of b200_block_qr_worksize bytes.  npc.qr uses it for real blocks of up to 384 rows and columns
 * (np_conserved.QR_HOUSEHOLDER_MAX).
 * Range: every finite block.  Each block is factored as 2^-e A_i, 2^e the power of two of max |a_ij| (exact), and R is
 * scaled back by 2^e: Q is bit for bit that of 2^-e A_i and R exactly 2^e times its R (rounded once where it is subnormal).
 * A pivot column of 2^-e A_i whose norm from the diagonal down is below 2^-450 is negligible: it gets no reflector, and
 * its entries below the diagonal (and the imaginary part of its diagonal entry) are dropped, so that columns many
 * orders of magnitude below the largest one cannot make Q non-orthogonal or non-finite. */
int64_t b200_block_qr_worksize(int64_t nblocks, const int64_t *m_host, const int64_t *n_host);
int b200_block_qr_f64(int64_t nblocks, const int64_t *m_host, const int64_t *n_host, const int64_t *a_off_host,
                      const int64_t *q_off_host, const int64_t *r_off_host, const double *A, double *Q, double *R,
                      void *work, int64_t work_bytes, b200_stream_t stream);

/* OUT[o, n, i] = sum_k M[n, k] T[o, k, i]  (T: outer x K x inner, OUT: outer x N x inner, row-major, i contiguous;
 * M: N x K on the device, K <= 32): a small matrix applied to the middle index without changing the layout.  Fuses the
 * two block transpositions and the skinny GEMM npc.tensordot needs for "W0.W1 applied to LP.theta" in the split-order
 * matvec (TwoSiteH.matvec, reference mps_common.py:1341-1343) into one streaming pass (taken for dense tensors with
 * K <= 32, SplitOrderMatvec._apply_W01_fused). */
int b200_mid_contract_f64(int64_t K, int64_t N, int64_t outer, int64_t inner, const double *M_dev, const double *T,
                          double *OUT, b200_stream_t stream);
/* two-segment version: [OUT1; OUT2][o, n, i] = sum_k M[n, k] [T1; T2][o, k, i] with K = K1 + K2 rows taken from T1 then
 * T2 and N = N1 + N2 rows written to OUT1 then OUT2 (M: N x K).  The matvec without the identity components of the
 * environments in one pass: T1 = LP_rest.theta, T2 = theta, OUT1 -> contraction with RP_rest, OUT2 -> added to the result. */
int b200_mid_contract2_f64(int64_t K1, int64_t K2, int64_t N1, int64_t N2, int64_t outer, int64_t inner,
                           const double *M_dev, const double *T1, const double *T2, double *OUT1, double *OUT2,
                           b200_stream_t stream);
/* complex two-segment version, the same contraction for complex M, T1, T2 in one read of each input.  M (N x K), T1
 * (outer x K1 x inner), T2 (outer x K2 x inner) and OUT2 (outer x N2 x inner) are planar: the real plane, then the
 * imaginary plane of the same size, in one buffer.  OUT1 is written as the real 2x2 embedding [[Yr, -Yi], [Yi, Yr]]
 * (2m x 2w, row-major) of the matrix Y[(o, n / C1), (n % C1, i)], m = outer N1 / C1, w = C1 inner: it is the left
 * operand of the next GEMM, which then multiplies the stacked planes [Br; Bi] of its right operand and returns a planar
 * result.  Serves the split-order matvec of complex states in the reference's combine=False contraction order
 * (mps_common.py:1340): T1 = LP_rest.theta, T2 = theta, OUT1 -> product with RP_rest, OUT2 -> added to the result.
 * Refused (B200_ERR_ARG): K = K1 + K2 outside 1..32, N = N1 + N2 above 1024, C1 not dividing N1 > 0, or both planes of M
 * above 48 KB. */
int b200_mid_contract2_z(int64_t K1, int64_t K2, int64_t N1, int64_t N2, int64_t C1, int64_t outer, int64_t inner,
                         const double *M_dev, const double *T1, const double *T2, double *OUT1, double *OUT2,
                         b200_stream_t stream);

/* OUT[c] = sum_r X[r*ld + c]^2 for a row-major (rows x cols) matrix (leverage scores of the null-space
 * completion in np_conserved.svd; no reference counterpart: LAPACK returns a complete basis by itself) */
int b200_col_sqnorms_f64(int64_t rows, int64_t cols, int64_t ld, const double *X, double *OUT,
                         b200_stream_t stream);

/* ---- block-diagonal SVD / eigh ------------------------------------------------------------------- */
/* Batched one-sided block-Jacobi SVD of nblocks independent row-major matrices A_i (m[i] x n[i]) at
 * a_off[i]: A_i = U_i diag(S_i) VT_i with k_i = min(m_i, n_i), S_i sorted descending,
 * U_i (m_i x k_i) at u_off[i], S_i at s_off[i], VT_i (k_i x n_i) at vt_off[i], all row-major.
 * A is not modified.  work_dev must hold b200_block_svd_worksize(...) bytes.  Synchronous on `stream`.
 * info_host[i] = number of Jacobi sweeps used (>0) or -1 if not converged.
 * Numerically negligible directions (row norm <= 16 eps sqrt(max(m,n)) |A_i|_F, i.e. singular values that are
 * zero to working precision) are deflated: their singular value is reported as found (tiny), the vector on the
 * accumulated side is exact (orthonormal), the vector on the other side is left ZERO and must be filled with an
 * orthonormal completion by the caller when it is needed (tenpy_b200.linalg.np_conserved.svd does).
 * nact_host[i] (may be NULL) = number of significant directions (they come first), transposed_host[i] (may be
 * NULL) = 1 if the zero vectors are columns of U_i, 0 if they are rows of VT_i.
 * Range: every finite block.  The iteration runs on 2^-e A_i, 2^e the power of two of max |a_ij| (exact): U, VT, nact
 * and transposed are bit for bit those of 2^-e A_i, S is exactly 2^e times its S (rounded once where it is subnormal).
 * The rotation criteria take square roots separately where a product of Gram entries under- or overflows, and row norms
 * whose plain sum of squares falls below 2^-900 are summed again rescaled, so rows graded far below the block's largest
 * entry neither stall the iteration nor lose their norm.  With deflation off (b200_svd_set_deflation(0)), rows whose
 * squared norm in the scaled block is at most 2^-990 (about 1e-149 max |a_ij|) are left unrotated: their Gram entries
 * are below the resolution of double precision.  With deflation on they lie far below the threshold anyway.
 * replaces _svd_worker npc:4950 -> svd_robust.svd svd_robust.py:37 (LAPACK gesdd / gesvd). */
/* switch the deflation of negligible directions in b200_block_svd_f64 on (default) / off; returns the old value */
int b200_svd_set_deflation(int on);
/* pivot eigen-solver of the real Jacobi rounds: 1 = jacobi_eig_kernel<false> (G in shared memory, three barriers per
 * rotation set), 3 = jacobi_eig_kernel_v3 (G and Q in registers, warp shuffles, two barriers per set); complex rounds
 * always use jacobi_eig_kernel<true>.  Returns the old value */
int b200_svd_set_eig_variant(int variant);
/* inner sweeps of the version-3 pivot eigen-solver (1..16, default 2): profiles/jacobi_sweeps_study.md finds the number
 * of outer sweeps unchanged between 2 and 4.  0 = "cross" mode: one pass over the pairs between the two row blocks of a
 * pivot only, the pairs inside a block once per outer sweep (the element-wise cyclic sweep in block order).  Returns the
 * old value */
int b200_svd_set_eig_inner_sweeps(int n);
/* small-block regime of the block SVD / eigh: while the longest row (columns of Y, rows of W) of the matrices still being
 * iterated is <= max_ld, a Jacobi round is ONE launch (jacobi_round_fused_kernel: Gram matrix, pivot eigen-solver and
 * both applications back to back in the CTA of the pair) instead of three with column splits.  Default 256
 * (environment B200_SVD_FUSED_LD); 0 switches the regime off.  Returns the old value */
int b200_svd_set_fused_max_ld(int max_ld);
/* additional deflation threshold relative to |A_i|_F (default 0 = rounding level only): directions with a
 * singular value below tol_rel*|A_i|_F are treated like the negligible ones; returns the old value.  A DMRG
 * truncation discards them anyway (the reference's `svd_min`, truncation.py:196). */
double b200_svd_set_deflation_tol(double tol_rel);
int64_t b200_block_svd_worksize(int64_t nblocks, const int64_t *m_host, const int64_t *n_host);
int b200_block_svd_f64(int64_t nblocks, const int64_t *m_host, const int64_t *n_host,
                       const int64_t *a_off_host, const int64_t *u_off_host, const int64_t *s_off_host,
                       const int64_t *vt_off_host, const double *A, double *U, double *S, double *VT,
                       void *work_dev, int64_t work_bytes, int32_t *info_host, int32_t *nact_host,
                       int32_t *transposed_host, b200_stream_t stream);
/* Complex counterpart of b200_block_svd_f64: A_i = U_i diag(S_i) VT_i for complex row-major blocks, with the same
 * shapes, offsets, ordering (S real, descending), synchronous call, info_host, sweep limit and deflation contract
 * (b200_svd_set_deflation / _set_deflation_tol apply).  PLANAR data: the real and imaginary parts are separate f64
 * buffers that share one offset table (A_re / A_im at a_off[i], U_re / U_im at u_off[i], VT_re / VT_im at vt_off[i]).
 * One-sided block Jacobi in complex arithmetic (Gram matrix P P^H, complex 2x2 rotations, real FP64 tensor-core products
 * on the planes); no block-size limit.  Rank-deficient blocks: as in the real entry, the vectors of the negligible
 * directions on the non-accumulated side are left ZERO (nact_host / transposed_host say which); the caller completes them
 * (tenpy_b200.linalg.np_conserved.svd does it with b200_block_qr_z).  Never produces NaN for finite input.  Range and
 * power-of-two scaling of the block: as b200_block_svd_f64 (max over the real and imaginary parts).
 * replaces _svd_worker npc:4950 -> svd_robust.svd (LAPACK zgesdd / zgesvd) for complex blocks. */
int64_t b200_block_svd_z_worksize(int64_t nblocks, const int64_t *m_host, const int64_t *n_host);
int b200_block_svd_z(int64_t nblocks, const int64_t *m_host, const int64_t *n_host, const int64_t *a_off_host,
                     const int64_t *u_off_host, const int64_t *s_off_host, const int64_t *vt_off_host,
                     const double *A_re, const double *A_im, double *U_re, double *U_im, double *S, double *VT_re,
                     double *VT_im, void *work_dev, int64_t work_bytes, int32_t *info_host, int32_t *nact_host,
                     int32_t *transposed_host, b200_stream_t stream);
/* Complex counterpart of b200_block_qr_f64: Householder QR (zgeqr2 + zung2r) of complex row-major blocks, planar buffers
 * sharing one offset table; Q_i (m_i x k_i) with orthonormal columns, R_i (k_i x n_i) upper triangular with a real
 * non-negative diagonal.  The same kernel and argument checks as b200_block_qr_f64, run with the imaginary planes.  One
 * CTA per block, one launch, every block size (cost O(m n k) on one SM: meant for the canonical-form path, not for large
 * dense blocks).  replaces the per-block np.linalg.qr of npc.qr (np_conserved.py:4139) for complex blocks.  `work` =
 * device scratch of b200_block_qr_z_worksize bytes (more than b200_block_qr_worksize of the same shapes).  Range and
 * power-of-two scaling of the block: as b200_block_qr_f64 (max over the real and imaginary parts). */
int64_t b200_block_qr_z_worksize(int64_t nblocks, const int64_t *m_host, const int64_t *n_host);
int b200_block_qr_z(int64_t nblocks, const int64_t *m_host, const int64_t *n_host, const int64_t *a_off_host,
                    const int64_t *q_off_host, const int64_t *r_off_host, const double *A_re, const double *A_im,
                    double *Q_re, double *Q_im, double *R_re, double *R_im, void *work, int64_t work_bytes,
                    b200_stream_t stream);

/* Batched symmetric eigen-decomposition of nblocks row-major symmetric matrices A_i (n[i] x n[i]):
 * A_i = V_i diag(W_i) V_i^T, W_i ascending, eigenvectors in the COLUMNS of V_i (row-major n x n).
 * Range: every finite block.  The iteration runs on 2^-e A_i, 2^e the power of two of max |a_ij| (exact): V is bit for
 * bit that of 2^-e A_i, W exactly 2^e times its W (rounded once where it is subnormal).  Accuracy |A_i|_F-normwise.
 * replaces _eig_worker npc:5041 (np.linalg.eigh, LAPACK syevd). */
int64_t b200_block_eigh_worksize(int64_t nblocks, const int64_t *n_host);
int b200_block_eigh_f64(int64_t nblocks, const int64_t *n_host, const int64_t *a_off_host,
                        const int64_t *w_off_host, const int64_t *v_off_host, const double *A, double *W,
                        double *V, void *work_dev, int64_t work_bytes, int32_t *info_host,
                        b200_stream_t stream);
/* Complex counterpart of b200_block_eigh_f64: A_i = V_i diag(W_i) V_i^H for complex Hermitian row-major blocks, with the
 * same shapes, offsets, synchronous call, info_host, sweep limit and error codes.  PLANAR data: A_re / A_im and V_re /
 * V_im are separate f64 buffers that share one offset table (a_off[i], v_off[i]); W_i is real and ascending, V_i unitary
 * with the eigenvectors in its COLUMNS: A_i V_i = V_i diag(W_i).  The iteration sees (A_i + A_i^H) / 2, as a Hermitian
 * solver reading one triangle would.  Range: every finite block.  The iteration runs on 2^-e A_i, 2^e the power of two of
 * max |a_ij| over the real and imaginary parts (exact): V is bit for bit that of 2^-e A_i, W exactly 2^e times its W
 * (rounded once where it is subnormal).  Accuracy |A_i|_F-normwise.
 * replaces _eig_worker npc:5041 (np.linalg.eigh, LAPACK zheevd) for complex blocks. */
int64_t b200_block_eigh_z_worksize(int64_t nblocks, const int64_t *n_host);
int b200_block_eigh_z(int64_t nblocks, const int64_t *n_host, const int64_t *a_off_host, const int64_t *w_off_host,
                      const int64_t *v_off_host, const double *A_re, const double *A_im, double *W, double *V_re,
                      double *V_im, void *work_dev, int64_t work_bytes, int32_t *info_host, b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200NPC_H */
