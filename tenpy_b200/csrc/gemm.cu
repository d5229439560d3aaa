// gemm.cu -- contraction plans (host) and the grouped FP64 tensor-core GEMM (device).
//
// Replaces, on the GPU, the reference's `_tensordot_worker` (tenpy/linalg/_npc_helper.pyx:1498):
//   * plan construction  <- _tensordot_pre_sort pyx:1337, _tensordot_match_charges pyx:1382,
//                           packing loop pyx:1710-1754 (host, integers only, cached by the caller)
//   * grouped GEMM       <- CblasGemmBatch.run pyx:204-274 (level-wise dgemm_batch).  Here every output
//                           tile owns its whole k-sum (all block pairs of its C block), so there is no
//                           beta=1 read-modify-write pass and no atomics.
#include <algorithm>
#include <cstdarg>
#include <cstring>
#include <numeric>
#include <vector>

#include "common.cuh"

namespace b200 {

thread_local std::string g_last_error;
std::atomic<long long> g_kernel_launches{0};

int set_error(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

int sm_count() {
    static int cached = -1;
    if (cached < 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess)
            cached = n;
        else
            return 132;
    }
    return cached;
}

// ---- device-side descriptors ---------------------------------------------------------------------
struct GemmTask {
    int64_t c_off;
    int32_t m, n;
    int32_t pair_begin, pair_end;
};
struct GemmPair {
    int64_t a_off, b_off;
    int32_t k, pad;
};
struct GemmTile {
    int32_t task, tm, tn, pad;
};

constexpr int GEMM_BK = 16;
constexpr int GEMM_STAGES = 3;

template <int BM, int BN>
constexpr int gemm_smem_bytes() {
    return GEMM_STAGES * (BM * (GEMM_BK + 4) + GEMM_BK * (BN + 4)) * (int)sizeof(double);
}

// One CTA computes one BM x BN tile of one output block, summing over all (A,B) block pairs of that
// output block.  cp.async 3-stage pipeline global->shared, DMMA m16n8k8 from shared, guarded epilogue.
// VEC: all row strides are even and all block bases 16-byte aligned -> 16-byte cp.async / stores.
template <int BM, int BN, int WARPS_M, int WARPS_N, bool VEC>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32)
    grouped_gemm_kernel(const double *__restrict__ A, const double *__restrict__ B, double *__restrict__ C,
                        const GemmTile *__restrict__ tiles, const GemmTask *__restrict__ tasks,
                        const GemmPair *__restrict__ pairs) {
    constexpr int BK = GEMM_BK, STAGES = GEMM_STAGES;
    constexpr int NTHR = WARPS_M * WARPS_N * 32;
    constexpr int WM = BM / WARPS_M, WN = BN / WARPS_N;
    constexpr int MT = WM / 16, NTL = WN / 8;
    constexpr int LDA_S = BK + 4, LDB_S = BN + 4;
    static_assert(WM % 16 == 0 && WN % 8 == 0, "warp tile");

    extern __shared__ __align__(16) double smem[];
    double *As = smem;
    double *Bs = smem + STAGES * BM * LDA_S;

    const GemmTile tile = tiles[blockIdx.x];
    const GemmTask task = tasks[tile.task];
    const int m = task.m, n = task.n;
    const int row0 = tile.tm * BM, col0 = tile.tn * BN;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int warp_m = warp / WARPS_N, warp_n = warp % WARPS_N;
    const int g = lane >> 2, t = lane & 3;

    // total number of k-steps over all pairs
    int total = 0;
    for (int p = task.pair_begin; p < task.pair_end; ++p) total += (pairs[p].k + BK - 1) / BK;

    // producer cursor
    int pp = task.pair_begin, pk = 0;
    GemmPair cur = (pp < task.pair_end) ? pairs[pp] : GemmPair{0, 0, 0, 0};   // a task without pairs writes zeros

    auto load_stage = [&](int stage) {
        const int k = cur.k;
        const int kbase = pk * BK;
        double *as = As + stage * BM * LDA_S;
        double *bs = Bs + stage * BK * LDB_S;
        const double *ag = A + cur.a_off;
        const double *bg = B + cur.b_off;
        if (VEC) {
            // A: BM rows x 8 chunks of 2 doubles
            constexpr int ACH = BM * (BK / 2);
#pragma unroll
            for (int c = tid; c < ACH; c += NTHR) {
                int r = c / (BK / 2), cc = (c % (BK / 2)) * 2;
                int gr = row0 + r, gc = kbase + cc;
                bool ok = (gr < m) && (gc < k);
                const double *src = ok ? (ag + (int64_t)gr * k + gc) : ag;
                cp_async16(as + r * LDA_S + cc, src, ok ? 16 : 0);
            }
            constexpr int BCH = BK * (BN / 2);
#pragma unroll
            for (int c = tid; c < BCH; c += NTHR) {
                int r = c / (BN / 2), cc = (c % (BN / 2)) * 2;
                int gr = kbase + r, gc = col0 + cc;
                bool ok = (gr < k) && (gc < n);
                const double *src = ok ? (bg + (int64_t)gr * n + gc) : bg;
                cp_async16(bs + r * LDB_S + cc, src, ok ? 16 : 0);
            }
        } else {
            constexpr int ACH = BM * BK;
#pragma unroll 4
            for (int c = tid; c < ACH; c += NTHR) {
                int r = c / BK, cc = c % BK;
                int gr = row0 + r, gc = kbase + cc;
                bool ok = (gr < m) && (gc < k);
                const double *src = ok ? (ag + (int64_t)gr * k + gc) : ag;
                cp_async8(as + r * LDA_S + cc, src, ok ? 8 : 0);
            }
            constexpr int BCH = BK * BN;
#pragma unroll 4
            for (int c = tid; c < BCH; c += NTHR) {
                int r = c / BN, cc = c % BN;
                int gr = kbase + r, gc = col0 + cc;
                bool ok = (gr < k) && (gc < n);
                const double *src = ok ? (bg + (int64_t)gr * n + gc) : bg;
                cp_async8(bs + r * LDB_S + cc, src, ok ? 8 : 0);
            }
        }
        // advance cursor
        ++pk;
        if (pk * BK >= k) {
            pk = 0;
            ++pp;
            if (pp < task.pair_end) cur = pairs[pp];
        }
    };

    double acc[MT][NTL][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NTL; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

    int loaded = 0;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (loaded < total) {
            load_stage(s);
            ++loaded;
        }
        cp_async_commit();
    }

    for (int it = 0; it < total; ++it) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        if (loaded < total) {
            load_stage((it + STAGES - 1) % STAGES);
            ++loaded;
        }
        cp_async_commit();

        const double *as = As + (it % STAGES) * BM * LDA_S + (warp_m * WM) * LDA_S;
        const double *bs = Bs + (it % STAGES) * BK * LDB_S + warp_n * WN;
#pragma unroll
        for (int kk = 0; kk < BK; kk += 8) {
            double af[MT][4], bf[NTL][2];
#pragma unroll
            for (int i = 0; i < MT; ++i) {
                const double *ap = as + (i * 16 + g) * LDA_S + kk + t;
                af[i][0] = ap[0];
                af[i][1] = ap[8 * LDA_S];
                af[i][2] = ap[4];
                af[i][3] = ap[8 * LDA_S + 4];
            }
#pragma unroll
            for (int j = 0; j < NTL; ++j) {
                const double *bp = bs + (kk + t) * LDB_S + j * 8 + g;
                bf[j][0] = bp[0];
                bf[j][1] = bp[4 * LDB_S];
            }
#pragma unroll
            for (int i = 0; i < MT; ++i)
#pragma unroll
                for (int j = 0; j < NTL; ++j) dmma_16x8x8(acc[i][j], af[i], bf[j]);
        }
    }
    cp_async_wait<0>();

    // epilogue
    double *cg = C + task.c_off;
#pragma unroll
    for (int i = 0; i < MT; ++i) {
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            int r = row0 + warp_m * WM + i * 16 + g;
            int c = col0 + warp_n * WN + j * 8 + 2 * t;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                int rr = r + 8 * h;
                if (rr < m) {
                    double *dst = cg + (int64_t)rr * n + c;
                    if (VEC) {
                        if (c < n) *reinterpret_cast<double2 *>(dst) = make_double2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
                    } else {
                        if (c < n) dst[0] = acc[i][j][2 * h];
                        if (c + 1 < n) dst[1] = acc[i][j][2 * h + 1];
                    }
                }
            }
        }
    }
}

// ---- thin block products: streaming kernels ---------------------------------------------------------------------------
// Contractions over an un-bunched MPO leg (LP.W0 -> LHeff, W1.RP -> RHeff, reference mpo.py:3107-3126) are lists of block
// products with k = 1 per pair, a handful of pairs per output block and ONE narrow side (n or m of a few elements), the
// other side being chi_sector^2 long.  A 32 x 32 tensor-core tile computes ~3 % useful work there and the launch has
// > 10^6 CTAs.  They are HBM-bound sums of a few scaled
// vectors: one thread per element of the long side, the narrow operand read through the read-only path (same address
// for the whole warp), coalesced on the long operand.
constexpr int THIN_MAX = 8;      // narrow side <= THIN_MAX elements
constexpr int THIN_KSUM = 64;    // sum of k over the pairs of the output block
constexpr int THIN_ROWS = 256;   // elements of the long side per CTA

// C (m x n), n <= THIN_MAX:  C[r, :] = sum_p sum_kk A_p[r, kk] B_p[kk, :]
__global__ void __launch_bounds__(THIN_ROWS)
    thin_n_kernel(const double *__restrict__ A, const double *__restrict__ B, double *__restrict__ C,
                  const GemmTile *__restrict__ tiles, const GemmTask *__restrict__ tasks, const GemmPair *__restrict__ pairs) {
    const GemmTile tile = tiles[blockIdx.x];
    const GemmTask task = tasks[tile.task];
    const int64_t r = (int64_t)tile.tm * THIN_ROWS + threadIdx.x;
    if (r >= task.m) return;
    const int n = task.n;
    double acc[THIN_MAX];
#pragma unroll
    for (int j = 0; j < THIN_MAX; ++j) acc[j] = 0.0;
    for (int p = task.pair_begin; p < task.pair_end; ++p) {
        const GemmPair pr = pairs[p];
        const double *a = A + pr.a_off + r * pr.k;
        const double *b = B + pr.b_off;
        for (int kk = 0; kk < pr.k; ++kk) {
            const double av = a[kk];
#pragma unroll
            for (int j = 0; j < THIN_MAX; ++j)
                if (j < n) acc[j] = fma(av, __ldg(b + (int64_t)kk * n + j), acc[j]);
        }
    }
    double *c = C + task.c_off + r * n;
#pragma unroll
    for (int j = 0; j < THIN_MAX; ++j)
        if (j < n) c[j] = acc[j];
}

// C (m x n), m <= THIN_MAX:  C[:, c] = sum_p sum_kk A_p[:, kk] B_p[kk, c]
__global__ void __launch_bounds__(THIN_ROWS)
    thin_m_kernel(const double *__restrict__ A, const double *__restrict__ B, double *__restrict__ C,
                  const GemmTile *__restrict__ tiles, const GemmTask *__restrict__ tasks, const GemmPair *__restrict__ pairs) {
    const GemmTile tile = tiles[blockIdx.x];
    const GemmTask task = tasks[tile.task];
    const int64_t col = (int64_t)tile.tn * THIN_ROWS + threadIdx.x;
    if (col >= task.n) return;
    const int m = task.m, n = task.n;
    double acc[THIN_MAX];
#pragma unroll
    for (int i = 0; i < THIN_MAX; ++i) acc[i] = 0.0;
    for (int p = task.pair_begin; p < task.pair_end; ++p) {
        const GemmPair pr = pairs[p];
        const double *a = A + pr.a_off;
        const double *b = B + pr.b_off + col;
        for (int kk = 0; kk < pr.k; ++kk) {
            const double bv = b[(int64_t)kk * n];
#pragma unroll
            for (int i = 0; i < THIN_MAX; ++i)
                if (i < m) acc[i] = fma(__ldg(a + (int64_t)i * pr.k + kk), bv, acc[i]);
        }
    }
    double *c = C + task.c_off + col;
#pragma unroll
    for (int i = 0; i < THIN_MAX; ++i)
        if (i < m) c[(int64_t)i * n] = acc[i];
}

// ---- host side: tiling of a task list --------------------------------------------------------------
struct TileSet {
    std::vector<GemmTile> tiles[5];  // 0: 128x128, 1: 64x64, 2: 32x32 (tensor core); 3: thin n, 4: thin m (streaming)
};

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

static void build_tiles(const std::vector<GemmTask> &tasks, const std::vector<GemmPair> &pairs, TileSet &ts) {
    struct Key {
        int64_t work;
        GemmTile tile;
    };
    std::vector<Key> keyed[5];
    static const int force_cfg = getenv("B200_GEMM_FORCE_CFG") ? atoi(getenv("B200_GEMM_FORCE_CFG")) : -1;
    for (size_t ti = 0; ti < tasks.size(); ++ti) {
        const GemmTask &tk = tasks[ti];
        if (tk.m <= 0 || tk.n <= 0) continue;
        int64_t ksum = 0;
        for (int p = tk.pair_begin; p < tk.pair_end; ++p) ksum += pairs[p].k;
        int64_t area128 = cdiv(tk.m, 128) * cdiv(tk.n, 128) * 128 * 128;
        int64_t area64 = cdiv(tk.m, 64) * cdiv(tk.n, 64) * 64 * 64;
        int64_t area32 = cdiv(tk.m, 32) * cdiv(tk.n, 32) * 32 * 32;
        // 64x64 tiles (4 warps, 4 CTAs/SM) are the default: more resident warps to cover the DMMA latency than
        // 128x128 (8 warps, 1 CTA/SM); the H100 runs the chi=1024 matvec products on them at 32-41 TFLOP/s (CUDA
        // events, H100 SXM 80 GB, 700 W).  The 128x128 kernel stays reachable through B200_GEMM_FORCE_CFG=0.
        (void)area128;
        int cfg = 1;
        if (area32 * 10 < area64 * 7) cfg = 2;
        if (force_cfg >= 0) cfg = force_cfg;   // tuning knob (environment B200_GEMM_FORCE_CFG)
        // thin products (one side <= THIN_MAX, short k-sum, long other side): streaming kernels
        if (force_cfg < 0 && ksum <= THIN_KSUM) {
            if (tk.n <= THIN_MAX && tk.m >= 4 * tk.n) cfg = 3;
            else if (tk.m <= THIN_MAX && tk.n >= 4 * tk.m) cfg = 4;
        }
        if (cfg >= 3) {
            int64_t nt = cdiv(cfg == 3 ? tk.m : tk.n, THIN_ROWS);
            for (int64_t i = 0; i < nt; ++i) {
                Key k;
                k.work = ksum;
                k.tile = cfg == 3 ? GemmTile{(int32_t)ti, (int32_t)i, 0, 0} : GemmTile{(int32_t)ti, 0, (int32_t)i, 0};
                keyed[cfg].push_back(k);
            }
            continue;
        }
        int b = cfg == 0 ? 128 : (cfg == 1 ? 64 : 32);
        for (int tm = 0; tm < cdiv(tk.m, b); ++tm)
            for (int tn = 0; tn < cdiv(tk.n, b); ++tn) {
                Key k;
                k.work = ksum;
                k.tile = GemmTile{(int32_t)ti, tm, tn, 0};
                keyed[cfg].push_back(k);
            }
    }
    for (int c = 0; c < 5; ++c) {
        std::stable_sort(keyed[c].begin(), keyed[c].end(), [](const Key &x, const Key &y) { return x.work > y.work; });
        ts.tiles[c].clear();
        for (auto &k : keyed[c]) ts.tiles[c].push_back(k.tile);
    }
}

struct DeviceGemmDesc {
    GemmTask *tasks = nullptr;
    GemmPair *pairs = nullptr;
    GemmTile *tiles[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    int n_tiles[5] = {0, 0, 0, 0, 0};
    bool vec = false;
    int device = -1;
    void release() {
        if (tasks) cudaFree(tasks);
        if (pairs) cudaFree(pairs);
        for (int c = 0; c < 5; ++c) {
            if (tiles[c]) cudaFree(tiles[c]);
            tiles[c] = nullptr;
        }
        tasks = nullptr;
        pairs = nullptr;
    }
};

static int upload_desc(const std::vector<GemmTask> &tasks, const std::vector<GemmPair> &pairs, DeviceGemmDesc &d) {
    TileSet ts;
    build_tiles(tasks, pairs, ts);
    B200_CUDA_CHECK(cudaGetDevice(&d.device));
    if (!tasks.empty()) {
        B200_CUDA_CHECK(cudaMalloc(&d.tasks, tasks.size() * sizeof(GemmTask)));
        B200_CUDA_CHECK(cudaMemcpy(d.tasks, tasks.data(), tasks.size() * sizeof(GemmTask), cudaMemcpyHostToDevice));
    }
    if (!pairs.empty()) {
        B200_CUDA_CHECK(cudaMalloc(&d.pairs, pairs.size() * sizeof(GemmPair)));
        B200_CUDA_CHECK(cudaMemcpy(d.pairs, pairs.data(), pairs.size() * sizeof(GemmPair), cudaMemcpyHostToDevice));
    }
    for (int c = 0; c < 5; ++c) {
        d.n_tiles[c] = (int)ts.tiles[c].size();
        if (d.n_tiles[c]) {
            B200_CUDA_CHECK(cudaMalloc(&d.tiles[c], ts.tiles[c].size() * sizeof(GemmTile)));
            B200_CUDA_CHECK(cudaMemcpy(d.tiles[c], ts.tiles[c].data(), ts.tiles[c].size() * sizeof(GemmTile),
                                       cudaMemcpyHostToDevice));
        }
    }
    // 16-byte vector path: every row stride even, every block offset even
    bool vec = true;
    for (auto &t : tasks)
        if ((t.n & 1) || (t.c_off & 1)) vec = false;
    for (auto &p : pairs)
        if ((p.k & 1) || (p.a_off & 1) || (p.b_off & 1)) vec = false;
    d.vec = vec;
    return B200_OK;
}

template <int BM, int BN, int WMW, int WNW, bool VEC>
static int launch_cfg(const DeviceGemmDesc &d, int cfg, const double *A, const double *B, double *C, cudaStream_t st) {
    if (d.n_tiles[cfg] == 0) return B200_OK;
    auto kern = grouped_gemm_kernel<BM, BN, WMW, WNW, VEC>;
    constexpr int smem = gemm_smem_bytes<BM, BN>();
    static bool attr_set = false;
    if (!attr_set) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_set = true;
    }
    kern<<<d.n_tiles[cfg], WMW * WNW * 32, smem, st>>>(A, B, C, d.tiles[cfg], d.tasks, d.pairs);
    B200_CHECK_LAUNCH();
    return B200_OK;
}

static int run_desc(const DeviceGemmDesc &d, const double *A, const double *B, double *C, cudaStream_t st) {
    int rc;
    if (d.n_tiles[3]) {
        thin_n_kernel<<<d.n_tiles[3], THIN_ROWS, 0, st>>>(A, B, C, d.tiles[3], d.tasks, d.pairs);
        B200_CHECK_LAUNCH();
    }
    if (d.n_tiles[4]) {
        thin_m_kernel<<<d.n_tiles[4], THIN_ROWS, 0, st>>>(A, B, C, d.tiles[4], d.tasks, d.pairs);
        B200_CHECK_LAUNCH();
    }
    if (d.vec && (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) == 0) {
        if ((rc = launch_cfg<128, 128, 2, 4, true>(d, 0, A, B, C, st))) return rc;
        if ((rc = launch_cfg<64, 64, 2, 2, true>(d, 1, A, B, C, st))) return rc;
        if ((rc = launch_cfg<32, 32, 2, 2, true>(d, 2, A, B, C, st))) return rc;
    } else {
        if ((rc = launch_cfg<128, 128, 2, 4, false>(d, 0, A, B, C, st))) return rc;
        if ((rc = launch_cfg<64, 64, 2, 2, false>(d, 1, A, B, C, st))) return rc;
        if ((rc = launch_cfg<32, 32, 2, 2, false>(d, 2, A, B, C, st))) return rc;
    }
    return B200_OK;
}

}  // namespace b200

using namespace b200;

// ---- plan object ---------------------------------------------------------------------------------
struct b200_tdot_plan {
    int32_t rank_c = 0;
    std::vector<int64_t> c_qdata, c_off, c_rows, c_cols;
    std::vector<GemmTask> tasks;
    std::vector<GemmPair> pairs;
    int64_t c_size = 0;
    double flops = 0.0;
    DeviceGemmDesc dev;
    bool uploaded = false;
};

namespace {
// compare rows of width w with the LAST column as primary key (np.lexsort(rows.T) order)
struct LexLess {
    const int64_t *base;
    int64_t stride;
    int32_t col0, w;
    bool operator()(int64_t i, int64_t j) const {
        const int64_t *x = base + i * stride + col0, *y = base + j * stride + col0;
        for (int32_t c = w - 1; c >= 0; --c) {
            if (x[c] != y[c]) return x[c] < y[c];
        }
        return false;
    }
    bool equal(int64_t i, int64_t j) const {
        const int64_t *x = base + i * stride + col0, *y = base + j * stride + col0;
        for (int32_t c = 0; c < w; ++c)
            if (x[c] != y[c]) return false;
        return true;
    }
};

// assign group ids (in lex order) to the rows of a table restricted to columns [col0, col0+w)
void group_ids(const int64_t *tab, int64_t n, int64_t stride, int32_t col0, int32_t w, std::vector<int64_t> &ids,
               std::vector<int64_t> &rep) {
    ids.assign(n, 0);
    rep.clear();
    if (n == 0) return;
    std::vector<int64_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    LexLess less{tab, stride, col0, w};
    if (w > 0) std::stable_sort(order.begin(), order.end(), less);
    int64_t gid = -1;
    for (int64_t i = 0; i < n; ++i) {
        if (i == 0 || (w > 0 && !less.equal(order[i - 1], order[i]))) {
            ++gid;
            rep.push_back(order[i]);
        }
        ids[order[i]] = gid;
    }
}
}  // namespace

extern "C" int b200_tdot_plan_create(const int64_t *a_qdata, int64_t n_a, int32_t rank_a, const int64_t *b_qdata,
                                     int64_t n_b, int32_t rank_b, int32_t n_contr, const int64_t *a_rows,
                                     const int64_t *a_cols, const int64_t *a_off, const int64_t *b_rows,
                                     const int64_t *b_cols, const int64_t *b_off, b200_tdot_plan **plan_out) {
    if (!plan_out) return set_error(B200_ERR_ARG, "plan_out is NULL");
    if (n_contr < 0 || n_contr > rank_a || n_contr > rank_b) return set_error(B200_ERR_ARG, "bad n_contr");
    const int32_t keep_a = rank_a - n_contr, keep_b = rank_b - n_contr;
    auto *plan = new b200_tdot_plan();
    plan->rank_c = keep_a + keep_b;

    // row groups of a (kept legs = first keep_a columns), column groups of b (kept = last keep_b columns)
    std::vector<int64_t> row_id, row_rep, col_id, col_rep;
    group_ids(a_qdata, n_a, rank_a, 0, keep_a, row_id, row_rep);
    group_ids(b_qdata, n_b, rank_b, n_contr, keep_b, col_id, col_rep);

    // ids of the contracted qindex tuples, shared between a and b
    std::vector<int64_t> contr(((size_t)n_a + n_b) * (n_contr > 0 ? n_contr : 1));
    for (int64_t i = 0; i < n_a; ++i)
        for (int32_t c = 0; c < n_contr; ++c) contr[i * n_contr + c] = a_qdata[i * rank_a + keep_a + c];
    for (int64_t j = 0; j < n_b; ++j)
        for (int32_t c = 0; c < n_contr; ++c) contr[(n_a + j) * n_contr + c] = b_qdata[j * rank_b + c];
    std::vector<int64_t> kid, krep;
    group_ids(contr.data(), n_a + n_b, n_contr > 0 ? n_contr : 1, 0, n_contr, kid, krep);
    const int64_t n_k = (int64_t)krep.size();

    // bucket blocks of b by contracted id
    std::vector<std::vector<int64_t>> b_by_k(n_k);
    for (int64_t j = 0; j < n_b; ++j) b_by_k[kid[n_a + j]].push_back(j);

    struct Prod {
        int64_t col, row, k, ai, bj;
    };
    std::vector<Prod> prods;
    for (int64_t i = 0; i < n_a; ++i) {
        const auto &bl = b_by_k[kid[i]];
        for (int64_t j : bl) {
            if (a_cols[i] != b_rows[j]) {
                delete plan;
                return set_error(B200_ERR_ARG, "contracted block sizes differ: a block %lld has k=%lld, b block %lld has k=%lld",
                                 (long long)i, (long long)a_cols[i], (long long)j, (long long)b_rows[j]);
            }
            prods.push_back(Prod{col_id[j], row_id[i], kid[i], i, j});
        }
    }
    std::sort(prods.begin(), prods.end(), [](const Prod &x, const Prod &y) {
        if (x.col != y.col) return x.col < y.col;
        if (x.row != y.row) return x.row < y.row;
        return x.k < y.k;
    });

    int64_t off = 0;
    for (size_t p = 0; p < prods.size(); ++p) {
        const Prod &pr = prods[p];
        bool new_task = (p == 0) || prods[p - 1].col != pr.col || prods[p - 1].row != pr.row;
        if (new_task) {
            GemmTask t;
            t.m = (int32_t)a_rows[pr.ai];
            t.n = (int32_t)b_cols[pr.bj];
            t.c_off = off;
            t.pair_begin = (int32_t)plan->pairs.size();
            t.pair_end = t.pair_begin;
            plan->tasks.push_back(t);
            plan->c_off.push_back(off);
            plan->c_rows.push_back(t.m);
            plan->c_cols.push_back(t.n);
            for (int32_t c = 0; c < keep_a; ++c) plan->c_qdata.push_back(a_qdata[pr.ai * rank_a + c]);
            for (int32_t c = 0; c < keep_b; ++c) plan->c_qdata.push_back(b_qdata[pr.bj * rank_b + n_contr + c]);
            int64_t sz = (int64_t)t.m * t.n;
            off += cdiv(sz, B200_BLOCK_ALIGN) * B200_BLOCK_ALIGN;
        }
        GemmTask &t = plan->tasks.back();
        if (a_rows[pr.ai] != t.m || b_cols[pr.bj] != t.n) {
            delete plan;
            return set_error(B200_ERR_ARG, "inconsistent block sizes within an output block");
        }
        // an empty product (zero-size contracted block) contributes nothing and must not take a pipeline stage of
        // grouped_gemm_kernel; its output block stays (a block with no products left is written as zeros)
        if (a_cols[pr.ai] <= 0) continue;
        GemmPair gp;
        gp.a_off = a_off[pr.ai];
        gp.b_off = b_off[pr.bj];
        gp.k = (int32_t)a_cols[pr.ai];
        gp.pad = 0;
        plan->pairs.push_back(gp);
        t.pair_end = (int32_t)plan->pairs.size();
        plan->flops += 2.0 * (double)t.m * (double)t.n * (double)gp.k;
    }
    plan->c_size = off;
    *plan_out = plan;
    return B200_OK;
}

extern "C" int b200_tdot_plan_info(const b200_tdot_plan *plan, int64_t *n_c, int64_t *n_pairs, int64_t *c_size,
                                   double *flops) {
    if (!plan) return set_error(B200_ERR_ARG, "plan is NULL");
    if (n_c) *n_c = (int64_t)plan->tasks.size();
    if (n_pairs) *n_pairs = (int64_t)plan->pairs.size();
    if (c_size) *c_size = plan->c_size;
    if (flops) *flops = plan->flops;
    return B200_OK;
}

extern "C" int b200_tdot_plan_get(const b200_tdot_plan *plan, int64_t *c_qdata, int64_t *c_off, int64_t *c_rows,
                                  int64_t *c_cols) {
    if (!plan) return set_error(B200_ERR_ARG, "plan is NULL");
    size_t n = plan->tasks.size();
    if (c_qdata && !plan->c_qdata.empty()) memcpy(c_qdata, plan->c_qdata.data(), plan->c_qdata.size() * sizeof(int64_t));
    if (c_off && n) memcpy(c_off, plan->c_off.data(), n * sizeof(int64_t));
    if (c_rows && n) memcpy(c_rows, plan->c_rows.data(), n * sizeof(int64_t));
    if (c_cols && n) memcpy(c_cols, plan->c_cols.data(), n * sizeof(int64_t));
    return B200_OK;
}

extern "C" int b200_tdot_plan_pairs(const b200_tdot_plan *plan, int64_t *pair_ptr, int64_t *a_off, int64_t *b_off,
                                    int64_t *k) {
    if (!plan) return set_error(B200_ERR_ARG, "plan is NULL");
    for (size_t t = 0; t < plan->tasks.size(); ++t) {
        pair_ptr[t] = plan->tasks[t].pair_begin;
        pair_ptr[t + 1] = plan->tasks[t].pair_end;
    }
    if (plan->tasks.empty()) pair_ptr[0] = 0;
    for (size_t p = 0; p < plan->pairs.size(); ++p) {
        a_off[p] = plan->pairs[p].a_off;
        b_off[p] = plan->pairs[p].b_off;
        k[p] = plan->pairs[p].k;
    }
    return B200_OK;
}

extern "C" int b200_tdot_plan_run(b200_tdot_plan *plan, const double *A, const double *B, double *C,
                                  b200_stream_t stream) {
    if (!plan) return set_error(B200_ERR_ARG, "plan is NULL");
    if (plan->tasks.empty()) return B200_OK;
    if (!plan->uploaded) {
        int rc = upload_desc(plan->tasks, plan->pairs, plan->dev);
        if (rc) return rc;
        plan->uploaded = true;
    }
    return run_desc(plan->dev, A, B, C, (cudaStream_t)stream);
}

extern "C" void b200_tdot_plan_destroy(b200_tdot_plan *plan) {
    if (!plan) return;
    if (plan->uploaded) plan->dev.release();
    delete plan;
}

extern "C" int b200_grouped_gemm_f64(int64_t n_tasks, const int64_t *m, const int64_t *n, const int64_t *c_off,
                                     const int64_t *pair_ptr, int64_t n_pairs, const int64_t *k, const int64_t *a_off,
                                     const int64_t *b_off, const double *A, const double *B, double *C,
                                     b200_stream_t stream) {
    if (n_tasks <= 0) return B200_OK;
    if (pair_ptr[n_tasks] > n_pairs) return set_error(B200_ERR_ARG, "grouped_gemm: pair_ptr exceeds n_pairs");
    std::vector<GemmTask> tasks((size_t)n_tasks);
    std::vector<GemmPair> pairs;
    pairs.reserve((size_t)n_pairs);
    for (int64_t t = 0; t < n_tasks; ++t) {
        tasks[t].c_off = c_off[t];
        tasks[t].m = (int32_t)m[t];
        tasks[t].n = (int32_t)n[t];
        tasks[t].pair_begin = (int32_t)pairs.size();
        for (int64_t p = pair_ptr[t]; p < pair_ptr[t + 1]; ++p) {
            if (k[p] <= 0) continue;   // an empty product contributes nothing (and must not take a pipeline stage)
            GemmPair pr;
            pr.a_off = a_off[p];
            pr.b_off = b_off[p];
            pr.k = (int32_t)k[p];
            pr.pad = 0;
            pairs.push_back(pr);
        }
        tasks[t].pair_end = (int32_t)pairs.size();   // a task without products writes a zero block
    }
    if (pairs.empty()) pairs.push_back(GemmPair{0, 0, 0, 0});   // (never dereferenced by a k-step; keeps the copies below non-empty)
    // descriptors go to a persistent grow-only device scratch (no cudaMalloc/cudaFree per call)
    static char *scratch = nullptr;
    static size_t scratch_cap = 0;
    static int scratch_dev = -1;
    TileSet ts;
    build_tiles(tasks, pairs, ts);
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    const size_t b_tasks = al(tasks.size() * sizeof(GemmTask)), b_pairs = al(pairs.size() * sizeof(GemmPair));
    size_t b_tiles[5], total = b_tasks + b_pairs;
    for (int c = 0; c < 5; ++c) {
        b_tiles[c] = al(ts.tiles[c].size() * sizeof(GemmTile));
        total += b_tiles[c];
    }
    int dev = 0;
    B200_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev != scratch_dev || total > scratch_cap) {
        if (scratch && dev == scratch_dev) cudaFree(scratch);
        scratch_cap = std::max<size_t>(total * 2, (size_t)1 << 20);
        B200_CUDA_CHECK(cudaMalloc(&scratch, scratch_cap));
        scratch_dev = dev;
    }
    cudaStream_t st = (cudaStream_t)stream;
    static cudaStream_t scratch_stream = nullptr;
    static bool scratch_used = false;
    if (scratch_used && scratch_stream != st) B200_CUDA_CHECK(cudaStreamSynchronize(scratch_stream));
    scratch_stream = st;
    scratch_used = true;
    DeviceGemmDesc d;
    d.device = dev;
    char *at = scratch;
    d.tasks = reinterpret_cast<GemmTask *>(at);
    B200_CUDA_CHECK(cudaMemcpyAsync(at, tasks.data(), tasks.size() * sizeof(GemmTask), cudaMemcpyHostToDevice, st));
    at += b_tasks;
    d.pairs = reinterpret_cast<GemmPair *>(at);
    B200_CUDA_CHECK(cudaMemcpyAsync(at, pairs.data(), pairs.size() * sizeof(GemmPair), cudaMemcpyHostToDevice, st));
    at += b_pairs;
    for (int c = 0; c < 5; ++c) {
        d.n_tiles[c] = (int)ts.tiles[c].size();
        d.tiles[c] = reinterpret_cast<GemmTile *>(at);
        if (d.n_tiles[c])
            B200_CUDA_CHECK(cudaMemcpyAsync(at, ts.tiles[c].data(), ts.tiles[c].size() * sizeof(GemmTile),
                                            cudaMemcpyHostToDevice, st));
        at += b_tiles[c];
    }
    bool vec = true;
    for (auto &t : tasks)
        if ((t.n & 1) || (t.c_off & 1)) vec = false;
    for (auto &p : pairs)
        if ((p.k & 1) || (p.a_off & 1) || (p.b_off & 1)) vec = false;
    d.vec = vec;
    // No host synchronisation: the pageable staging vectors are consumed by cudaMemcpyAsync before it returns, and the next
    // call's copies into `scratch` are ordered behind this call's kernels as long as both use the same stream (a call on
    // another stream waits for the previous one first, see above).
    return run_desc(d, A, B, C, st);
}

// ---- misc ABI ------------------------------------------------------------------------------------
extern "C" int64_t b200_kernel_launch_count(int reset) {
    long long v = reset ? g_kernel_launches.exchange(0) : g_kernel_launches.load();
    return (int64_t)v;
}
extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }
extern "C" const char *b200_last_error(void) { return g_last_error.c_str(); }
extern "C" int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}
extern "C" int b200_device_info(int dev, int *sm, int *cc_major, int *cc_minor, int64_t *mem_bytes) {
    cudaDeviceProp prop;
    B200_CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    if (sm) *sm = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    if (mem_bytes) *mem_bytes = (int64_t)prop.totalGlobalMem;
    return B200_OK;
}
