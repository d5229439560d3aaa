// Host check of tenpy_b200/csrc/block_qr_core.cuh (test infrastructure): the phases of block_qr_kernel are run for
// tid = 0..T-1 sequentially, exactly as the CUDA kernel runs them between barriers; checks A = Q R, Q^T Q = 1, R upper
// triangular with non-negative diagonal, on tall / wide / square / rank deficient / zero-column blocks; then power-of-two
// equivariance: the QR of 2^e A must give Q bit for bit and R = 2^e R(A) exactly for every e that keeps 2^e A normal.
// Run by tests/test_host_qr_scale.py.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "../../tenpy_b200/csrc/block_qr_core.cuh"

using namespace b200::bqr;
constexpr int T = 256;

// A (in) -> R (out, first k rows), as block_qr_kernel
static void qr_emulated(std::vector<double> &A_io, std::vector<double> &Q, int m, int n) {
    const int k = std::min(m, n);
    std::vector<double> A((size_t)m * n), V((size_t)m * k, 0.0), partial(T), params(3), taus(k), sign(k);
    for (int t = 0; t < T; ++t) absmax_partial(t, T, A_io.data(), nullptr, (int64_t)m * n, partial.data());
    const double scale = block_scale(T, partial.data()), rscale = 1.0 / scale;
    for (int t = 0; t < T; ++t) scale_in(t, T, A_io.data(), A.data(), (int64_t)m * n, scale);
    for (int j = 0; j < k; ++j) {
        for (int t = 0; t < T; ++t) col_partial(t, T, A.data(), m, n, j, partial.data());
        reflector(T, A.data(), n, j, partial.data(), params.data());                          // thread 0
        taus[j] = params[0];
        for (int t = 0; t < T; ++t) store_reflector(t, T, A.data(), V.data(), m, n, k, j, params.data());
        for (int t = 0; t < T; ++t) apply_reflector(t, T, A.data(), n, V.data(), m, k, j, j + 1, taus[j]);
    }
    for (int t = 0; t < T; ++t) init_q(t, T, Q.data(), m, k);
    for (int j = k - 1; j >= 0; --j)
        for (int t = 0; t < T; ++t) apply_reflector(t, T, Q.data(), k, V.data(), m, k, j, j, taus[j]);
    for (int t = 0; t < T; ++t) sign_of_diag(t, T, A.data(), n, k, sign.data());
    for (int t = 0; t < T; ++t) flip_signs(t, T, A.data(), Q.data(), m, n, k, sign.data());
    std::fill(A_io.begin(), A_io.end(), 0.0);                         // rows >= k: A_io's R part is k x n
    for (int t = 0; t < T; ++t) store_r(t, T, A.data(), A_io.data(), k, n, rscale);
}

// number of entries where x != 2^e y (NaN counts as a mismatch)
static int mismatches(const std::vector<double> &x, const std::vector<double> &y, int e, int len) {
    int bad = 0;
    for (int i = 0; i < len; ++i) bad += (x[i] == std::ldexp(y[i], e)) ? 0 : 1;
    return bad;
}

static int scale_cases(std::mt19937_64 &rng) {
    std::normal_distribution<double> nd(0.0, 1.0);
    std::uniform_int_distribution<int> small(-4, 4);
    const int exps[] = {-990, -700, -540, -520, -300, -270, -260, -80, 0, 80, 260, 270, 300, 511, 540, 700, 990};
    // {m, n, kind}: 0 = Gaussian with every |a| in [2^-30, 2^4] (2^e A normal for |e| <= 990), 1 = rank 5 with small
    // integer factors (exact zeros and exact rank deficiency), 2 = all zero
    const int blocks[][3] = {{40, 25, 0}, {25, 40, 0}, {33, 33, 0}, {30, 30, 1}, {12, 20, 1}, {6, 4, 2}};
    int bad = 0;
    for (auto &bl : blocks) {
        const int m = bl[0], n = bl[1], kind = bl[2], k = std::min(m, n);
        std::vector<double> A0((size_t)m * n, 0.0);
        if (kind == 0) {
            for (auto &a : A0) {
                const double x = nd(rng);
                a = std::copysign(std::min(std::max(std::fabs(x), std::ldexp(1.0, -30)), 15.0), x);
            }
        } else if (kind == 1) {
            std::vector<double> X((size_t)m * 5), Y((size_t)5 * n);
            for (auto &x : X) x = small(rng);
            for (auto &y : Y) y = small(rng);
            for (int i = 0; i < m; ++i)
                for (int j = 0; j < n; ++j)
                    for (int r = 0; r < 5; ++r) A0[(size_t)i * n + j] += X[(size_t)i * 5 + r] * Y[(size_t)r * n + j];
        }
        std::vector<double> R0 = A0, Q0((size_t)m * k, -5.0);
        qr_emulated(R0, Q0, m, n);
        for (int e : exps) {
            std::vector<double> R((size_t)m * n), Q((size_t)m * k, -5.0);
            for (size_t i = 0; i < R.size(); ++i) R[i] = std::ldexp(A0[i], e);
            qr_emulated(R, Q, m, n);
            const int bq = mismatches(Q, Q0, 0, m * k), br = mismatches(R, R0, e, k * n);
            if (bq || br) {
                printf("scale 2^%d: %d x %d kind %d: %d entries of Q differ, %d of 2^-e R\n", e, m, n, kind, bq, br);
                ++bad;
            }
        }
    }
    printf("scale cases: %s\n", bad ? "FAILED" : "ok");
    return bad;
}

int main() {
    std::mt19937_64 rng(11);
    std::normal_distribution<double> nd(0.0, 1.0);
    const int shapes[][3] = {{7, 4, 0}, {4, 7, 0}, {5, 5, 0}, {1, 3, 0}, {3, 1, 0}, {33, 20, 0}, {64, 64, 0}, {300, 17, 0},
                             {12, 8, 3}, {40, 40, 10}, {9, 6, -1}, {1, 1, 0}};
    int bad = 0;
    for (auto &sh : shapes) {
        const int m = sh[0], n = sh[1], rank = sh[2], k = std::min(m, n);
        std::vector<double> A0((size_t)m * n);
        if (rank > 0) {                                   // rank deficient: product of thin factors
            std::vector<double> X((size_t)m * rank), Y((size_t)rank * n);
            for (auto &x : X) x = nd(rng);
            for (auto &y : Y) y = nd(rng);
            for (int i = 0; i < m; ++i)
                for (int j = 0; j < n; ++j) {
                    double s = 0.0;
                    for (int r = 0; r < rank; ++r) s += X[(size_t)i * rank + r] * Y[(size_t)r * n + j];
                    A0[(size_t)i * n + j] = s;
                }
        } else {
            for (auto &a : A0) a = nd(rng);
            if (rank < 0)                                 // an exactly zero column
                for (int i = 0; i < m; ++i) A0[(size_t)i * n + 2] = 0.0;
        }
        std::vector<double> R = A0, Q((size_t)m * k, -5.0);
        qr_emulated(R, Q, m, n);
        double rec = 0.0, orth = 0.0, low = 0.0, mindiag = 1e300, amax = 0.0;
        for (auto a : A0) amax = std::max(amax, std::fabs(a));
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < n; ++j) {
                double s = 0.0;
                for (int c = 0; c < k; ++c) s += Q[(size_t)i * k + c] * R[(size_t)c * n + j];
                rec = std::max(rec, std::fabs(s - A0[(size_t)i * n + j]));
            }
        for (int a = 0; a < k; ++a)
            for (int b = 0; b < k; ++b) {
                double s = 0.0;
                for (int i = 0; i < m; ++i) s += Q[(size_t)i * k + a] * Q[(size_t)i * k + b];
                orth = std::max(orth, std::fabs(s - (a == b ? 1.0 : 0.0)));
            }
        for (int i = 0; i < k; ++i) {
            mindiag = std::min(mindiag, R[(size_t)i * n + i]);
            for (int j = 0; j < i && j < n; ++j) low = std::max(low, std::fabs(R[(size_t)i * n + j]));
        }
        printf("%3d x %3d rank %2d: |QR-A| %.2e  |QtQ-1| %.2e  lower %.1e  min diag %.2e\n", m, n, rank, rec / std::max(amax, 1e-300),
               orth, low, mindiag);
        if (!(rec <= 1e-13 * std::max(amax, 1e-300) * std::max(m, n)) || !(orth < 1e-13) || low != 0.0 || !(mindiag >= 0.0)) ++bad;
    }
    bad += scale_cases(rng);
    printf("%s\n", bad ? "FAILED" : "ok");
    return bad ? 1 : 0;
}
