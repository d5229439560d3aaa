// Host check of tenpy_b200/csrc/block_qr_core.cuh (test infrastructure): the phases of block_qr_kernel are run for
// tid = 0..T-1 sequentially, exactly as the CUDA kernel runs them between barriers, for real blocks and for complex blocks
// (imaginary planes filled); checks A = Q R, Q^H Q = 1, R upper triangular with a real non-negative diagonal, on tall /
// wide / square / rank deficient / zero-column blocks and blocks whose columns span 2^-1050 .. 2^1000; then power-of-two
// equivariance: the QR of 2^e A must give Q bit for bit and R = 2^e R(A) exactly for every e that keeps 2^e A normal.
// Run by tests/test_host_qr_scale.py.
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <random>
#include <vector>

#include "../../tenpy_b200/csrc/block_qr_core.cuh"

using namespace b200::bqr;
using cd = std::complex<double>;
constexpr int T = 256;

// A (in) -> R (out, first k rows), as block_qr_kernel; Ai_io / Qi: the imaginary planes of a complex block, else NULL
static void qr_emulated(std::vector<double> &A_io, std::vector<double> &Q, int m, int n, std::vector<double> *Ai_io,
                        std::vector<double> *Qi) {
    const int k = std::min(m, n);
    const bool cplx = Ai_io != nullptr;
    const int64_t mn = (int64_t)m * n;
    std::vector<double> A(mn), Ai(cplx ? mn : 0), V((size_t)m * k, 0.0), Vi(cplx ? (size_t)m * k : 0, 0.0), partial(T),
        params(5), taus(k), tausi(k), sign(k);
    const double *ai_in = cplx ? Ai_io->data() : nullptr;
    double *ai = cplx ? Ai.data() : nullptr, *vi = cplx ? Vi.data() : nullptr, *qi = cplx ? Qi->data() : nullptr;
    for (int t = 0; t < T; ++t) absmax_partial(t, T, A_io.data(), ai_in, mn, partial.data());
    const double scale = block_scale(T, partial.data()), rscale = 1.0 / scale;
    for (int t = 0; t < T; ++t) scale_in(t, T, A_io.data(), A.data(), mn, scale, ai_in, ai);
    for (int j = 0; j < k; ++j) {
        for (int t = 0; t < T; ++t) col_partial(t, T, A.data(), m, n, j, partial.data(), ai);
        reflector(T, A.data(), n, j, partial.data(), params.data(), ai);                       // thread 0
        taus[j] = params[0];
        tausi[j] = params[3];
        for (int t = 0; t < T; ++t) store_reflector(t, T, A.data(), V.data(), m, n, k, j, params.data(), ai, vi);
        for (int t = 0; t < T; ++t)
            apply_reflector(t, T, A.data(), n, V.data(), m, k, j, j + 1, taus[j], ai, vi, cplx ? -tausi[j] : 0.0);
    }
    for (int t = 0; t < T; ++t) init_q(t, T, Q.data(), m, k, qi);
    for (int j = k - 1; j >= 0; --j)
        for (int t = 0; t < T; ++t)
            apply_reflector(t, T, Q.data(), k, V.data(), m, k, j, j, taus[j], qi, vi, cplx ? tausi[j] : 0.0);
    for (int t = 0; t < T; ++t) sign_of_diag(t, T, A.data(), n, k, sign.data());
    for (int t = 0; t < T; ++t) flip_signs(t, T, A.data(), Q.data(), m, n, k, sign.data(), ai, qi);
    std::fill(A_io.begin(), A_io.end(), 0.0);                         // rows >= k: A_io's R part is k x n
    if (cplx) std::fill(Ai_io->begin(), Ai_io->end(), 0.0);
    for (int t = 0; t < T; ++t) store_r(t, T, A.data(), A_io.data(), k, n, rscale, ai, cplx ? Ai_io->data() : nullptr);
}

// the planes of a complex (or, with cplx false, real) block as the kernel takes them
static void split(const std::vector<cd> &X, std::vector<double> &re, std::vector<double> &im) {
    re.resize(X.size());
    im.resize(X.size());
    for (size_t i = 0; i < X.size(); ++i) {
        re[i] = X[i].real();
        im[i] = X[i].imag();
    }
}

// QR of the block X (m x n): R (k x n) and Q (m x k), both planes (imaginary parts zero for a real block)
static void qr_block(const std::vector<cd> &X, int m, int n, bool cplx, std::vector<double> &Rr, std::vector<double> &Ri,
                     std::vector<double> &Qr, std::vector<double> &Qi) {
    const int k = std::min(m, n);
    split(X, Rr, Ri);
    Qr.assign((size_t)m * k, -5.0);
    Qi.assign((size_t)m * k, cplx ? -5.0 : 0.0);
    qr_emulated(Rr, Qr, m, n, cplx ? &Ri : nullptr, cplx ? &Qi : nullptr);
}

// number of entries where x != 2^e y (NaN counts as a mismatch)
static int mismatches(const std::vector<double> &x, const std::vector<double> &y, int e, int len) {
    int bad = 0;
    for (int i = 0; i < len; ++i) bad += (x[i] == std::ldexp(y[i], e)) ? 0 : 1;
    return bad;
}

static int scale_cases(std::mt19937_64 &rng, bool cplx) {
    const char *tag = cplx ? "complex " : "";
    std::normal_distribution<double> nd(0.0, 1.0);
    std::uniform_int_distribution<int> small(-4, 4);
    const int exps[] = {-990, -700, -540, -520, -300, -270, -260, -80, 0, 80, 260, 270, 300, 511, 540, 700, 990};
    // {m, n, kind}: 0 = Gaussian with every |a| in [2^-30, 2^4] (2^e A normal for |e| <= 990), 1 = rank 5 with small
    // integer factors (exact zeros and exact rank deficiency), 2 = all zero; complex: both planes so
    const int blocks[][3] = {{40, 25, 0}, {25, 40, 0}, {33, 33, 0}, {30, 30, 1}, {12, 20, 1}, {6, 4, 2}};
    auto clamped = [&]() {
        const double x = nd(rng);
        return std::copysign(std::min(std::max(std::fabs(x), std::ldexp(1.0, -30)), 15.0), x);
    };
    auto small_entries = [&](std::vector<cd> &v) {
        for (auto &x : v) x = small(rng);
        if (cplx)
            for (auto &x : v) x += cd(0.0, small(rng));
    };
    int bad = 0;
    for (auto &bl : blocks) {
        const int m = bl[0], n = bl[1], kind = bl[2], k = std::min(m, n);
        std::vector<cd> A0((size_t)m * n, 0.0);
        if (kind == 0) {
            for (auto &a : A0) a = clamped();
            if (cplx)
                for (auto &a : A0) a += cd(0.0, clamped());
        } else if (kind == 1) {
            std::vector<cd> X((size_t)m * 5), Y((size_t)5 * n);
            small_entries(X);
            small_entries(Y);
            for (int i = 0; i < m; ++i)
                for (int j = 0; j < n; ++j)
                    for (int r = 0; r < 5; ++r) A0[(size_t)i * n + j] += X[(size_t)i * 5 + r] * Y[(size_t)r * n + j];
        }
        std::vector<double> R0, R0i, Q0, Q0i;
        qr_block(A0, m, n, cplx, R0, R0i, Q0, Q0i);
        for (int e : exps) {
            std::vector<cd> Ae(A0.size());
            for (size_t i = 0; i < Ae.size(); ++i) Ae[i] = cd(std::ldexp(A0[i].real(), e), std::ldexp(A0[i].imag(), e));
            std::vector<double> R, Ri, Q, Qi;
            qr_block(Ae, m, n, cplx, R, Ri, Q, Qi);
            const int bq = mismatches(Q, Q0, 0, m * k) + mismatches(Qi, Q0i, 0, m * k);
            const int br = mismatches(R, R0, e, k * n) + mismatches(Ri, R0i, e, k * n);
            if (bq || br) {
                printf("%sscale 2^%d: %d x %d kind %d: %d entries of Q differ, %d of 2^-e R\n", tag, e, m, n, kind, bq, br);
                ++bad;
            }
        }
    }
    printf("%sscale cases: %s\n", tag, bad ? "FAILED" : "ok");
    return bad;
}

static int shape_cases(std::mt19937_64 &rng, bool cplx) {
    std::normal_distribution<double> nd(0.0, 1.0);
    auto gaussian = [&](std::vector<cd> &v) {
        for (auto &x : v) x = nd(rng);
        if (cplx)
            for (auto &x : v) x += cd(0.0, nd(rng));
    };
    const int shapes[][3] = {{7, 4, 0}, {4, 7, 0}, {5, 5, 0}, {1, 3, 0}, {3, 1, 0}, {33, 20, 0}, {64, 64, 0}, {300, 17, 0},
                             {12, 8, 3}, {40, 40, 10}, {9, 6, -1}, {1, 1, 0}, {7, 5, -2}, {40, 30, -2}, {30, 40, -2}};
    int bad = 0;
    for (auto &sh : shapes) {
        const int m = sh[0], n = sh[1], rank = sh[2], k = std::min(m, n);
        std::vector<cd> A0((size_t)m * n);
        if (rank > 0) {                                   // rank deficient: product of thin factors
            std::vector<cd> X((size_t)m * rank), Y((size_t)rank * n);
            gaussian(X);
            gaussian(Y);
            for (int i = 0; i < m; ++i)
                for (int j = 0; j < n; ++j) {
                    cd s = 0.0;
                    for (int r = 0; r < rank; ++r) s += X[(size_t)i * rank + r] * Y[(size_t)r * n + j];
                    A0[(size_t)i * n + j] = s;
                }
        } else {
            gaussian(A0);
            if (rank == -1)                               // an exactly zero column
                for (int i = 0; i < m; ++i) A0[(size_t)i * n + 2] = 0.0;
            if (rank == -2) {                             // columns scaled by 2^1000 .. 2^-1050: after the block scaling
                const int col_exp[] = {1000, 480, -1050, 470, -25, 490, 0, 475, -537};   // squares subnormal or zero
                for (int i = 0; i < m; ++i)
                    for (int j = 0; j < n; ++j) {
                        const int e = col_exp[j % 9];
                        A0[(size_t)i * n + j] = cd(std::ldexp(A0[(size_t)i * n + j].real(), e),
                                                   std::ldexp(A0[(size_t)i * n + j].imag(), e));
                    }
            }
        }
        std::vector<double> Rr, Ri, Qr, Qi;
        qr_block(A0, m, n, cplx, Rr, Ri, Qr, Qi);
        auto R = [&](int i, int j) { return cd(Rr[(size_t)i * n + j], Ri[(size_t)i * n + j]); };
        auto Q = [&](int i, int j) { return cd(Qr[(size_t)i * k + j], Qi[(size_t)i * k + j]); };
        double rec = 0.0, orth = 0.0, low = 0.0, mindiag = 1e300, imdiag = 0.0, amax = 0.0;
        bool finite = true;
        for (size_t i = 0; i < Qr.size(); ++i) finite = finite && std::isfinite(Qr[i]) && std::isfinite(Qi[i]);
        for (size_t i = 0; i < Rr.size(); ++i) finite = finite && std::isfinite(Rr[i]) && std::isfinite(Ri[i]);
        for (auto a : A0) amax = std::max(amax, std::abs(a));
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < n; ++j) {
                cd s = 0.0;
                for (int c = 0; c < k; ++c) s += Q(i, c) * R(c, j);
                rec = std::max(rec, std::abs(s - A0[(size_t)i * n + j]));
            }
        for (int a = 0; a < k; ++a)
            for (int b = 0; b < k; ++b) {
                cd s = 0.0;
                for (int i = 0; i < m; ++i) s += std::conj(Q(i, a)) * Q(i, b);
                orth = std::max(orth, std::abs(s - (a == b ? 1.0 : 0.0)));
            }
        for (int i = 0; i < k; ++i) {
            mindiag = std::min(mindiag, R(i, i).real());
            imdiag = std::max(imdiag, std::fabs(R(i, i).imag()));
            for (int j = 0; j < i && j < n; ++j) low = std::max(low, std::abs(R(i, j)));
        }
        printf("%s%3d x %3d rank %2d: |QR-A| %.2e  |QtQ-1| %.2e  lower %.1e  min diag %.2e\n", cplx ? "complex " : "", m, n,
               rank, rec / std::max(amax, 1e-300), orth, low, mindiag);
        if (!finite || !(rec <= 1e-13 * std::max(amax, 1e-300) * std::max(m, n)) || !(orth < 1e-13) || low != 0.0 ||
            !(mindiag >= 0.0) || imdiag != 0.0)
            ++bad;
    }
    return bad;
}

int main() {
    std::mt19937_64 rng(11);
    int bad = 0;
    for (bool cplx : {false, true}) {
        bad += shape_cases(rng, cplx);
        bad += scale_cases(rng, cplx);
    }
    printf("%s\n", bad ? "FAILED" : "ok");
    return bad ? 1 : 0;
}
