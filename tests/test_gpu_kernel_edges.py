"""GPU tests of the C-ABI kernels at their edge shapes, against dense references.

Reference rules:
* products and reductions are compared with numpy in ``np.longdouble``; every bound is a constant (written next to the
  assert) times eps times the componentwise scale of the operation (``|A||B|``, ``sum |x_i y_i|``);
* data movement and ``scale_axis`` round once or not at all: they must match numpy exactly;
* output buffers are filled with NaN and the blocks laid out with gaps: every element outside the blocks must be untouched.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev(a):
    from tenpy_b200 import backend
    return backend.to_device(np.ascontiguousarray(a))


def _host(t):
    from tenpy_b200 import backend
    return backend.to_host(t).copy()


def _nan(n):
    import torch
    from tenpy_b200 import backend
    return torch.full((max(int(n), 1),), float('nan'), dtype=torch.float64, device=backend.device())


def _layout(rng, sizes, max_gap=5):
    """offsets of blocks of the given sizes laid out back to back with random gaps (>= 1 before every block)"""
    offs, at = [], 0
    for s in sizes:
        at += int(rng.integers(1, max_gap + 1))
        offs.append(at)
        at += int(s)
    return np.array(offs, dtype=np.int64), at + int(rng.integers(1, max_gap + 1))


def _assert_gaps_untouched(buf, offs, sizes):
    inside = np.zeros(len(buf), dtype=bool)
    for o, s in zip(offs, sizes):
        inside[o:o + s] = True
    assert np.all(np.isnan(buf[~inside])), 'a kernel wrote outside its blocks'


def _strided(buf, off, shape, strides):
    return np.lib.stride_tricks.as_strided(buf[off:], shape=tuple(int(s) for s in shape),
                                           strides=tuple(8 * int(s) for s in strides))


# ---- block QR -----------------------------------------------------------------------------------------------------------

def _qr_inputs(rng):
    mats = []
    for sh in [(1, 1), (1, 9), (13, 1), (57, 21), (21, 57), (40, 40), (384, 384), (384, 17), (17, 384)]:
        mats.append(('random %dx%d' % sh, rng.standard_normal(sh), True))
    mats.append(('zero', np.zeros((9, 6)), False))
    # upper triangular with a negative diagonal: every pivot column is zero below the diagonal (sigma == 0 in
    # bqr::reflector, tau = 0) and every R[j][j] needs the sign flip
    T = np.triu(rng.standard_normal((11, 7)))
    T[np.arange(7), np.arange(7)] = -1. - rng.random(7)
    mats.append(('zero column under a negative pivot', T, True))
    # one zero column inside a random block: sigma == 0 in the middle of the factorisation
    Z = rng.standard_normal((20, 12))
    Z[3:, 4] = 0.
    Z[4, 4] = -0.5
    mats.append(('zero column below a negative pivot inside', Z, False))
    mats.append(('rank 5', rng.standard_normal((30, 5)) @ rng.standard_normal((5, 23)), False))
    mats.append(('column-graded', rng.standard_normal((60, 25)) * np.logspace(0, -12, 25)[None, :], False))
    return mats


def test_block_qr_batch(gpu_lib):
    """b200_block_qr_f64 (npc.qr sends every real block <= np_conserved.QR_HOUSEHOLDER_MAX = 384 here) on one batch of
    edge shapes: Q^T Q = 1, R upper triangular with a non-negative diagonal, QR = A, and Q, R equal LAPACK's after the
    sign fix"""
    rng = np.random.default_rng(101)
    mats = _qr_inputs(rng)
    ms = [a.shape[0] for _, a, _ in mats]
    ns = [a.shape[1] for _, a, _ in mats]
    ks = [min(m, n) for m, n in zip(ms, ns)]
    a_off, a_len = _layout(rng, [m * n for m, n in zip(ms, ns)])
    q_off, q_len = _layout(rng, [m * k for m, k in zip(ms, ks)])
    r_off, r_len = _layout(rng, [k * n for k, n in zip(ks, ns)])
    A = np.full(a_len, np.nan)
    for (_, a, _), o in zip(mats, a_off):
        A[o:o + a.size] = a.ravel()
    dA, dQ, dR = _dev(A), _nan(q_len), _nan(r_len)
    gpu_lib.block_qr(ms, ns, a_off, q_off, r_off, dA, dQ, dR)
    Q, R = _host(dQ), _host(dR)
    assert np.array_equal(_host(dA), A, equal_nan=True)                  # input untouched
    _assert_gaps_untouched(Q, q_off, [m * k for m, k in zip(ms, ks)])
    _assert_gaps_untouched(R, r_off, [k * n for k, n in zip(ks, ns)])
    for (name, a, full_rank), m, n, k, qo, ro in zip(mats, ms, ns, ks, q_off, r_off):
        q = Q[qo:qo + m * k].reshape(m, k)
        r = R[ro:ro + k * n].reshape(k, n)
        c = 8 * max(m, n, 16)     # Householder QR: backward error and loss of orthogonality ~ max(m, n) eps
        assert np.max(np.abs(q.T @ q - np.eye(k))) <= c * EPS, name
        assert np.all(np.tril(r, -1) == 0.), name
        assert np.all(np.diag(r) >= 0.), name
        anorm = max(np.linalg.norm(a), 1e-300)
        assert np.linalg.norm(q.astype(LD) @ r.astype(LD) - a) <= c * EPS * anorm, name
        if full_rank:
            qr_, rr_ = np.linalg.qr(a)
            sgn = np.where(np.diag(rr_) < 0, -1., 1.)
            qr_, rr_ = qr_ * sgn[None, :], rr_ * sgn[:, None]
            cond = np.linalg.cond(a)
            # both factorisations are backward stable: the factors differ by ~ cond(A) max(m, n) eps
            assert np.max(np.abs(q - qr_)) <= c * EPS * cond, name
            assert np.max(np.abs(r - rr_)) <= c * EPS * cond * anorm, name
        if name == 'zero':
            assert np.array_equal(q, np.eye(m, k)) and np.all(r == 0.)


# ---- mid_contract / mid_contract2 ---------------------------------------------------------------------------------------

@pytest.mark.parametrize('K,N,outer,inner', [
    (1, 1, 3, 1), (12, 12, 5, 255), (16, 40, 2, 257), (17, 5, 4, 255), (32, 192, 2, 257),   # N K = 6144: 48 KB of M
    (1, 1024, 2, 3), (3, 2, 70001, 1)])                                                       # outer > 65535: grid-y loop
def test_mid_contract(gpu_lib, K, N, outer, inner):
    """OUT[o, n, i] = sum_k M[n, k] T[o, k, i] (KMAX = 16 for K <= 16, 32 above) against a long-double einsum; the output
    sits inside a NaN-filled buffer"""
    rng = np.random.default_rng(K * 1000 + N + outer)
    M = rng.standard_normal((N, K))
    T = rng.standard_normal((outer, K, inner))
    size, pad = outer * N * inner, 5
    buf = _nan(size + 2 * pad)
    gpu_lib.mid_contract(K, N, outer, inner, _dev(M), _dev(T), buf[pad:pad + size])
    out = _host(buf)
    _assert_gaps_untouched(out, [pad], [size])
    got = out[pad:pad + size].reshape(outer, N, inner)
    ref = np.einsum('nk,oki->oni', M.astype(LD), T.astype(LD))
    den = np.einsum('nk,oki->oni', np.abs(M), np.abs(T))
    assert np.all(np.abs(got - ref) <= (K + 1) * EPS * den)              # K chained FMAs


@pytest.mark.parametrize('K1,K2,N1,N2,outer,inner', [
    (5, 7, 6, 6, 3, 255), (0, 12, 4, 8, 2, 257), (12, 0, 9, 3, 2, 255), (3, 20, 0, 9, 2, 1), (16, 16, 96, 96, 2, 100),
    (9, 7, 10, 0, 3, 257), (1, 1, 1, 1, 1, 1), (4, 4, 2, 2, 66000, 1)])
def test_mid_contract2(gpu_lib, K1, K2, N1, N2, outer, inner):
    """the two-segment version, including empty K or N segments, against a long-double einsum of the stacked operands"""
    rng = np.random.default_rng(K1 * 100 + K2 * 10 + N1 + N2)
    K, N = K1 + K2, N1 + N2
    M = rng.standard_normal((N, K))
    T1 = rng.standard_normal((outer, K1, inner))
    T2 = rng.standard_normal((outer, K2, inner))
    s1, s2, pad = outer * N1 * inner, outer * N2 * inner, 3
    b1, b2 = _nan(s1 + 2 * pad), _nan(s2 + 2 * pad)
    gpu_lib.mid_contract2(K1, K2, N1, N2, outer, inner, _dev(M), _dev(T1.ravel() if K1 else np.zeros(1)),
                          _dev(T2.ravel() if K2 else np.zeros(1)), b1[pad:], b2[pad:])
    o1, o2 = _host(b1), _host(b2)
    _assert_gaps_untouched(o1, [pad], [s1])
    _assert_gaps_untouched(o2, [pad], [s2])
    T = np.concatenate([T1, T2], axis=1)
    ref = np.einsum('nk,oki->oni', M.astype(LD), T.astype(LD))
    den = np.einsum('nk,oki->oni', np.abs(M), np.abs(T))
    got = np.concatenate([o1[pad:pad + s1].reshape(outer, N1, inner), o2[pad:pad + s2].reshape(outer, N2, inner)], axis=1)
    assert np.all(np.abs(got - ref) <= (K + 1) * EPS * den)              # K chained FMAs


def test_mid_contract_argument_checks(gpu_lib):
    """K > 32, N > 1024 and an M above 48 KB are refused on the host (B200_ERR_ARG) before any launch"""
    from tenpy_b200._lib import B200Error
    M, T, OUT = _nan(64), _nan(64), _nan(64)
    for K, N in ((33, 1), (32, 193), (1, 1025)):
        with pytest.raises(B200Error, match='error 1:'):
            gpu_lib.mid_contract(K, N, 1, 1, M, T, OUT)
    for K1, K2, N1, N2 in ((17, 16, 1, 1), (16, 16, 100, 100), (0, 0, 1, 1), (-1, 2, 1, 1), (1, 1, 600, 425)):
        with pytest.raises(B200Error, match='error 1:'):
            gpu_lib.mid_contract2(K1, K2, N1, N2, 1, 1, M, T, T, OUT, OUT)
    assert np.all(np.isnan(_host(OUT)))


# ---- block moves --------------------------------------------------------------------------------------------------------

def _copy_tasks(rng, n_tasks, max_dim, big=None):
    """random strided copy records (rank 0..6): the source of every task is a sub-block of a larger C-contiguous array read
    with its axes permuted, the destination is contiguous"""
    recs, src_sizes, dst_sizes, tasks = [], [], [], []
    for t in range(n_tasks):
        rank = int(rng.integers(0, 7)) if big is None else len(big)
        sub = np.array(big if big is not None else rng.integers(1, max_dim + 1, rank), dtype=np.int64)
        full = sub + (rng.integers(0, 3, rank) if big is None else 0)
        cs = np.array([int(np.prod(full[d + 1:])) for d in range(rank)], dtype=np.int64)
        perm = rng.permutation(rank)
        shape = sub[perm]
        sstride = cs[perm]
        dstride = np.array([int(np.prod(shape[d + 1:])) for d in range(rank)], dtype=np.int64)
        tasks.append((shape, sstride, dstride))
        src_sizes.append(int(np.prod(full)))
        dst_sizes.append(int(np.prod(shape)))
    s_off, s_len = _layout(rng, src_sizes)
    d_off, d_len = _layout(rng, dst_sizes)
    for (shape, sstride, dstride), so, do, n in zip(tasks, s_off, d_off, dst_sizes):
        rec = np.zeros(22, dtype=np.int64)
        r = len(shape)
        rec[0], rec[1], rec[2], rec[3] = so, do, n, r
        rec[4:10] = 1
        rec[4:4 + r], rec[10:10 + r], rec[16:16 + r] = shape, sstride, dstride
        recs.append(rec)
    return np.array(recs), s_len, d_len, dst_sizes


@pytest.mark.parametrize('n_tasks,max_dim,big', [(64, 5, None), (3000, 3, None), (1, 0, (3, 517, 700)),
                                                 (2, 0, (2, 3, 5, 7, 11, 13))])
def test_copy_blocks(gpu_lib, n_tasks, max_dim, big):
    """strided N-d block copies of ranks 0..6 with random permutations and strides, thousands of small tasks in one launch,
    and a task of ~10^6 elements that spans many CTAs along x: exact, nothing written outside the destinations"""
    rng = np.random.default_rng(n_tasks + max_dim)
    recs, s_len, d_len, d_sizes = _copy_tasks(rng, n_tasks, max_dim, big)
    src = rng.standard_normal(s_len)
    dst = _nan(d_len)
    gpu_lib.copy_blocks(recs, _dev(recs), _dev(src), dst)
    got = _host(dst)
    exp = np.full(d_len, np.nan)
    for rec in recs:
        r = int(rec[3])
        shape = rec[4:4 + r]
        _strided(exp, rec[1], shape, rec[16:16 + r])[...] = _strided(src, rec[0], shape, rec[10:10 + r])
    assert np.array_equal(got, exp, equal_nan=True)
    _assert_gaps_untouched(got, recs[:, 1], d_sizes)


def test_take_blocks(gpu_lib):
    """take along the middle axis (Array.iproject): random sorted index sets, keep-all and keep-one, exact"""
    rng = np.random.default_rng(31)
    shapes = [(1, 1, 1), (3, 7, 5), (1, 300, 1), (40, 2, 33), (2, 1000, 260), (5, 9, 1), (7, 50, 3)]
    keeps = []
    for i, (o, l, _) in enumerate(shapes):
        if i % 3 == 0:
            keeps.append(np.arange(l))                                     # keep all
        elif i % 3 == 1:
            keeps.append(np.array([int(rng.integers(l))]))                 # keep one
        else:
            keeps.append(np.sort(rng.choice(l, size=int(rng.integers(1, l + 1)), replace=False)))
    s_off, s_len = _layout(rng, [o * l * i for o, l, i in shapes])
    d_sizes = [o * len(kp) * i for (o, _, i), kp in zip(shapes, keeps)]
    d_off, d_len = _layout(rng, d_sizes)
    i_off = np.concatenate(([0], np.cumsum([len(kp) for kp in keeps])[:-1])).astype(np.int64)
    idx = np.concatenate(keeps).astype(np.int64)
    recs = np.array([[so, do, o, len(kp), i, l, io] for (o, l, i), kp, so, do, io in zip(shapes, keeps, s_off, d_off, i_off)],
                    dtype=np.int64)
    src = rng.standard_normal(s_len)
    dst = _nan(d_len)
    gpu_lib.take_blocks(recs, _dev(recs), _dev(idx), _dev(src), dst)
    got = _host(dst)
    _assert_gaps_untouched(got, d_off, d_sizes)
    for (o, l, i), kp, so, do, n in zip(shapes, keeps, s_off, d_off, d_sizes):
        ref = np.take(src[so:so + o * l * i].reshape(o, l, i), kp, axis=1)
        assert np.array_equal(got[do:do + n].reshape(ref.shape), ref)


def test_scale_axis(gpu_lib):
    """x[o, j, i] *= s[j] over the first (outer = 1), a middle and the last axis (inner = 1): one rounding, exact"""
    rng = np.random.default_rng(32)
    shapes = [(1, 37, 50), (6, 11, 13), (40, 29, 1), (1, 1, 1), (3, 1000, 300), (1, 5, 1)]
    x_off, x_len = _layout(rng, [o * l * i for o, l, i in shapes])
    s_off = np.concatenate(([0], np.cumsum([l for _, l, _ in shapes])[:-1])).astype(np.int64) + 3
    S = rng.standard_normal(3 + sum(l for _, l, _ in shapes))
    X = np.full(x_len, np.nan)
    for (o, l, i), xo in zip(shapes, x_off):
        X[xo:xo + o * l * i] = rng.standard_normal(o * l * i)
    recs = np.array([[xo, o, l, i, so] for (o, l, i), xo, so in zip(shapes, x_off, s_off)], dtype=np.int64)
    dX = _dev(X)
    gpu_lib.scale_axis(recs, _dev(recs), _dev(S), dX)
    got = _host(dX)
    _assert_gaps_untouched(got, x_off, [o * l * i for o, l, i in shapes])
    for (o, l, i), xo, so in zip(shapes, x_off, s_off):
        ref = X[xo:xo + o * l * i].reshape(o, l, i) * S[so:so + l][None, :, None]
        assert np.array_equal(got[xo:xo + o * l * i].reshape(o, l, i), ref)


@pytest.mark.parametrize('rows,cols,ld', [(1, 1, 1), (37, 300, 311), (1000, 3, 4), (5, 257, 260), (0, 4, 4)])
def test_col_sqnorms(gpu_lib, rows, cols, ld):
    """column sums of squares of a row-major matrix with ld > cols (the padding columns are NaN and must not be read)"""
    rng = np.random.default_rng(rows + cols)
    X = np.full((max(rows, 1), ld), np.nan)
    X[:rows, :cols] = rng.standard_normal((rows, cols))
    out = _nan(cols + 3)
    gpu_lib.col_sqnorms(rows, cols, ld, _dev(X), out)
    got = _host(out)
    assert np.all(np.isnan(got[cols:]))
    ref = np.sum(X[:rows, :cols].astype(LD) ** 2, axis=0)
    assert np.all(np.abs(got[:cols] - ref) <= (rows + 1) * EPS * ref)   # `rows` chained FMAs


# ---- segment BLAS-1, dense BLAS-1 offsets, device-scalar Lanczos ----------------------------------------------------------

def _segments(rng, n_seg, lens):
    lens = np.asarray(lens, dtype=np.int64)
    x_off, x_len = _layout(rng, lens)
    order = rng.permutation(n_seg)                      # y holds the segments in another order, with other gaps
    y_off_sorted, y_len = _layout(rng, lens[order])
    y_off = np.empty(n_seg, dtype=np.int64)
    y_off[order] = y_off_sorted
    return np.stack([x_off, y_off, lens], axis=1), x_len, y_len


@pytest.mark.parametrize('case', ['many', 'long', 'mixed'])
def test_blas1_segments(gpu_lib, case):
    """axpy / dot over (x_off, y_off, len) segments: up to 2048 segments, lengths 0 .. ~10^6, x and y laid out differently"""
    from tenpy_b200 import backend
    rng = np.random.default_rng({'many': 1, 'long': 2, 'mixed': 3}[case])
    if case == 'many':
        lens = rng.integers(0, 400, 2048)
        lens[::97] = 0
    elif case == 'long':
        lens = np.array([1 << 20, 0, 999_983, 1, 5])
    else:
        lens = np.concatenate([rng.integers(0, 50, 500), [700_001, 0, 3]])
    n_seg = len(lens)
    seg, x_len, y_len = _segments(rng, n_seg, lens)
    X, Y = np.full(x_len, np.nan), np.full(y_len, np.nan)
    for xo, yo, n in seg:
        X[xo:xo + n] = rng.standard_normal(n)
        Y[yo:yo + n] = rng.standard_normal(n)
    dX, dY, dseg = _dev(X), _dev(Y), _dev(seg)
    out = backend.scalar_out()
    gpu_lib.dot_segments(n_seg, dseg, int(lens.max()), dX, dY, backend.dot_scratch(), out)
    got = backend.read_scalar(out)
    ref = sum(np.dot(X[xo:xo + n].astype(LD), Y[yo:yo + n].astype(LD)) for xo, yo, n in seg)
    den = sum(np.dot(np.abs(X[xo:xo + n]), np.abs(Y[yo:yo + n])) for xo, yo, n in seg)
    # per-thread FMA chains of <= max_len / 256 terms, then two tree reductions (< 64 levels)
    assert abs(got - ref) <= (lens.max() / 256 + 64) * EPS * den
    alpha = -0.7316
    gpu_lib.axpy_segments(n_seg, dseg, int(lens.max()), alpha, dX, dY)
    gY = _host(dY)
    _assert_gaps_untouched(gY, seg[:, 1], lens)
    for xo, yo, n in seg:
        ref = Y[yo:yo + n].astype(LD) + LD(alpha) * X[xo:xo + n].astype(LD)
        den = np.abs(Y[yo:yo + n]) + abs(alpha) * np.abs(X[xo:xo + n])
        assert np.all(np.abs(gY[yo:yo + n] - ref) <= 1 * EPS * den)      # one FMA: one rounding


@pytest.mark.parametrize('ox,oy', [(0, 0), (1, 1), (0, 1), (1, 0)])
@pytest.mark.parametrize('n', [1, 2, 7, 10, 4097, 1_000_001])
def test_blas1_offsets(gpu_lib, n, ox, oy):
    """axpy / scal / dot on views at element offsets 0 and 1 (16-byte vector branch or scalar branch) with odd and even n
    (the tail element of the vector branch); the elements around the view stay untouched; dot is deterministic"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(n + 10 * ox + 20 * oy)
    x, y = rng.standard_normal(n), rng.standard_normal(n)
    bx, by = _nan(n + 2), _nan(n + 2)
    bx[ox:ox + n] = _dev(x)
    by[oy:oy + n] = _dev(y)
    vx, vy = bx[ox:ox + n], by[oy:oy + n]
    out = backend.scalar_out()
    gpu_lib.dot(n, vx, vy, backend.dot_scratch(), out)
    d1 = backend.read_scalar(out)
    gpu_lib.dot(n, vx, vy, backend.dot_scratch(), out)
    assert np.float64(backend.read_scalar(out)).tobytes() == np.float64(d1).tobytes()   # same bits twice
    # per-thread chains of <= n / (256 * grid) terms (grid >= 1), two tree reductions
    assert abs(d1 - np.dot(x.astype(LD), y.astype(LD))) <= (n / 256 + 64) * EPS * np.dot(np.abs(x), np.abs(y))
    alpha = 0.3711
    gpu_lib.axpy(n, alpha, vx, vy)
    gy = _host(by)
    ref = y.astype(LD) + LD(alpha) * x.astype(LD)
    assert np.all(np.abs(gy[oy:oy + n] - ref) <= 1 * EPS * (np.abs(y) + alpha * np.abs(x)))   # one FMA: one rounding
    gpu_lib.scal(n, -1.37, vx)
    gx = _host(bx)
    assert np.array_equal(gx[ox:ox + n], x * -1.37)                      # one rounding, exact
    for g, o in ((gx, ox), (gy, oy)):
        assert np.all(np.isnan(np.delete(g, np.arange(o, o + n))))


@pytest.mark.parametrize('with_v0', [True, False])
@pytest.mark.parametrize('n', [1, 1000, 2 ** 20 + 3])
def test_lanczos_device_scalars_bitwise(gpu_lib, n, with_v0):
    """lanczos_update_dev (alpha from the device, beta = sqrt(beta2) on the device) is bit-identical to lanczos_update with
    the same alpha and sqrt(beta2) from the host, scal_rsqrt_dev to scal(1 / np.sqrt(n2)); both against long double"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(n + with_v0)
    w, v1, v0 = rng.standard_normal(n), rng.standard_normal(n), rng.standard_normal(n)
    dv1, dv0 = _dev(v1), _dev(v0)
    alpha_dev = backend.zeros(1)
    gpu_lib.dot(n, dv1, _dev(w), backend.dot_scratch(), alpha_dev)     # alpha as the Lanczos step makes it
    beta2 = float(rng.random()) * 3.
    beta2_dev = _dev(np.array([beta2]))
    alpha = backend.read_scalar(alpha_dev)
    beta = float(np.sqrt(beta2))
    dw_h, dw_d = _dev(w), _dev(w)
    out_h, out_d = backend.zeros(1), backend.zeros(1)
    scratch2 = backend.zeros(2048)
    gpu_lib.lanczos_update(n, alpha, dv1, beta, dv0 if with_v0 else None, dw_h, backend.dot_scratch(), out_h)
    gpu_lib.lanczos_update_dev(n, alpha_dev, dv1, beta2_dev if with_v0 else None, dv0 if with_v0 else None, dw_d,
                               scratch2, out_d)
    wh, wd = _host(dw_h), _host(dw_d)
    assert wh.tobytes() == wd.tobytes()
    assert _host(out_h).tobytes() == _host(out_d).tobytes()
    ref = w.astype(LD) - LD(alpha) * v1.astype(LD) - (LD(beta) * v0.astype(LD) if with_v0 else 0)
    den = np.abs(w) + abs(alpha) * np.abs(v1) + (beta * np.abs(v0) if with_v0 else 0)
    assert np.all(np.abs(wd - ref) <= 2 * EPS * den)                    # two FMAs: two roundings
    n2 = backend.read_scalar(out_d)
    assert abs(n2 - np.dot(wd.astype(LD), wd.astype(LD))) <= (n / 256 + 64) * EPS * np.dot(wd, wd)
    dx_h, dx_d = _dev(v1), _dev(v1)
    gpu_lib.scal(n, 1. / np.sqrt(n2), dx_h)
    gpu_lib.scal_rsqrt_dev(n, out_d, dx_d)
    assert _host(dx_h).tobytes() == _host(dx_d).tobytes()


# ---- contraction plans and the grouped GEMM -----------------------------------------------------------------------------

def _lexkey(t):
    return tuple(reversed(tuple(int(x) for x in t)))     # np.lexsort order: the LAST column is the primary key


def _plan_case(rng, keep_a, nc, keep_b, sizes, fill=0.6):
    """random block tables of a (keep_a kept legs, nc contracted) and b (nc contracted, keep_b kept); sizes[l] = block sizes
    of leg l (legs: a's kept, contracted, b's kept)"""
    import itertools
    la = sizes[:keep_a + nc]
    lb = sizes[keep_a:]

    def table(legs):
        rows = [t for t in itertools.product(*[range(len(s)) for s in legs]) if rng.random() < fill]
        return np.array(rows, dtype=np.int64).reshape(-1, len(legs))
    qa, qb = table(la), table(lb)

    def dims(q, legs, split):
        r = np.array([int(np.prod([legs[l][t[l]] for l in range(split)])) for t in q], dtype=np.int64)
        c = np.array([int(np.prod([legs[l][t[l]] for l in range(split, len(legs))])) for t in q], dtype=np.int64)
        return r, c
    a_rows, a_cols = dims(qa, la, keep_a)
    b_rows, b_cols = dims(qb, lb, nc)
    a_off, a_len = _layout(rng, a_rows * a_cols)
    b_off, b_len = _layout(rng, b_rows * b_cols)
    A, B = np.full(a_len, np.nan), np.full(b_len, np.nan)
    for o, r, c in zip(a_off, a_rows, a_cols):
        A[o:o + r * c] = rng.standard_normal(r * c)
    for o, r, c in zip(b_off, b_rows, b_cols):
        B[o:o + r * c] = rng.standard_normal(r * c)
    return qa, qb, a_rows, a_cols, a_off, b_rows, b_cols, b_off, A, B


@pytest.mark.parametrize('case', ['nc1', 'nc2', 'zero-k', 'zero-k-first'])
def test_tdot_plan(gpu_lib, case):
    """b200_tdot_plan_create + run on random block tables: the block table against a numpy block-sparse contraction,
    C against long double, the padding between the C blocks untouched, the product list without empty products.
    'zero-k-first': a zero-size contracted block (k = 0) ordered before non-empty ones in every output block."""
    rng = np.random.default_rng({'nc1': 1, 'nc2': 2, 'zero-k': 3, 'zero-k-first': 4}[case])
    if case == 'nc1':
        ka, nc, kb, sizes = 2, 1, 2, [[3, 5, 1], [2, 7], [4, 9, 17, 1], [6, 3], [11, 2, 5]]
    elif case == 'nc2':
        ka, nc, kb, sizes = 1, 2, 2, [[13, 5, 24], [2, 7, 1], [9, 17], [6, 33], [11, 20]]
    elif case == 'zero-k':
        ka, nc, kb, sizes = 2, 1, 1, [[3, 12], [2, 9], [5, 0, 20], [30, 4, 10]]
    else:
        ka, nc, kb, sizes = 1, 1, 1, [[20, 33], [0, 19, 40], [17, 24]]
    qa, qb, a_rows, a_cols, a_off, b_rows, b_cols, b_off, A, B = _plan_case(
        rng, ka, nc, kb, sizes, fill=1.0 if case == 'zero-k-first' else 0.6)
    plan = gpu_lib.tdot_plan(qa, qb, nc, a_rows, a_cols, a_off, b_rows, b_cols, b_off)
    # numpy: output blocks (row group of a, column group of b) with at least one common contracted tuple
    prods = {}
    for i, ta in enumerate(qa):
        for j, tb in enumerate(qb):
            if tuple(ta[ka:]) == tuple(tb[:nc]):
                prods.setdefault((tuple(ta[:ka]), tuple(tb[nc:])), []).append((_lexkey(ta[ka:]), i, j))
    keys = sorted(prods, key=lambda rc: (_lexkey(rc[1]), _lexkey(rc[0])))
    assert plan.n_c == len(keys)
    assert np.array_equal(plan.c_qdata, np.array([r + c for r, c in keys], dtype=np.int64).reshape(len(keys), ka + kb))
    rows = np.array([a_rows[prods[key][0][1]] for key in keys], dtype=np.int64)
    cols = np.array([b_cols[prods[key][0][2]] for key in keys], dtype=np.int64)
    sz = rows * cols
    c_off = np.concatenate(([0], np.cumsum((sz + 15) // 16 * 16)))
    assert np.array_equal(plan.c_rows, rows) and np.array_equal(plan.c_cols, cols)
    assert np.array_equal(plan.c_off, c_off[:-1]) and plan.c_size == c_off[-1]
    assert plan.flops == sum(2. * r * c * a_cols[i] for key, r, c in zip(keys, rows, cols) for _, i, _ in prods[key])
    C = _nan(plan.c_size)
    plan.run(_dev(A), _dev(B), C)
    C = _host(C)
    _assert_gaps_untouched(C, c_off[:-1], sz)
    for t, key in enumerate(keys):
        m, n = int(rows[t]), int(cols[t])
        ref = np.zeros((m, n), dtype=LD)
        den = np.zeros((m, n))
        ksum = 0
        for _, i, j in prods[key]:
            k = int(a_cols[i])
            a = A[a_off[i]:a_off[i] + m * k].reshape(m, k)
            b = B[b_off[j]:b_off[j] + k * n].reshape(k, n)
            ref += a.astype(LD) @ b.astype(LD)
            den += np.abs(a) @ np.abs(b)
            ksum += k
        got = C[c_off[t]:c_off[t] + m * n].reshape(m, n)
        assert np.all(np.abs(got - ref) <= (ksum + 1) * EPS * den), (case, t, key)   # one FMA chain of ksum terms
    # product list: the non-empty products of every output block, in the order of their contracted tuples
    pair_ptr, pa, pb, pk = plan.pairs()
    assert plan.n_pairs == len(pk) and pair_ptr[-1] == len(pk)
    for t, key in enumerate(keys):
        exp = [(a_off[i], b_off[j], a_cols[i]) for _, i, j in sorted(prods[key]) if a_cols[i] > 0]
        got = list(zip(pa[pair_ptr[t]:pair_ptr[t + 1]], pb[pair_ptr[t]:pair_ptr[t + 1]], pk[pair_ptr[t]:pair_ptr[t + 1]]))
        assert got == exp, (case, t)


@pytest.mark.parametrize('cfg', [0, 1, 2])
def test_grouped_gemm_forced_tiles(cfg):
    """test_grouped_gemm once more with every product on one tile configuration (B200_GEMM_FORCE_CFG, read once per
    process: 0 = 128 x 128, 1 = 64 x 64, 2 = 32 x 32, no thin kernels), in a child process that ends before this returns"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    env = dict(os.environ, B200_GEMM_FORCE_CFG=str(cfg), PYTHONDONTWRITEBYTECODE='1')
    flags = ['-s'] if sys.flags.no_user_site else []      # the child sees the same packages as this process
    res = subprocess.run([sys.executable] + flags + ['-m', 'pytest', '-q', '-p', 'no:cacheprovider', '-m', 'gpu',
                          os.path.join(ROOT, 'tests', 'test_gpu_kernels.py') + '::test_grouped_gemm',
                          os.path.join(ROOT, 'tests', 'test_gpu_kernels.py') + '::test_selftest'],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert ' passed' in res.stdout and 'skipped' not in res.stdout, res.stdout[-3000:]


# ---- SVD and eigh -------------------------------------------------------------------------------------------------------

def test_block_svd_zero_block(gpu_lib):
    """an all-zero block in a mixed batch is fully deflated (nact = 0, S = 0) and its accumulated side is orthonormal;
    the other blocks are unaffected"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(41)
    mats = [rng.standard_normal((20, 12)), np.zeros((15, 9)), rng.standard_normal((7, 30)), np.zeros((6, 6)),
            np.zeros((3, 40)), rng.standard_normal((33, 33))]
    shapes = [a.shape for a in mats]
    ks = [min(s) for s in shapes]
    a_off = np.concatenate(([0], np.cumsum([a.size for a in mats])[:-1]))
    u_off = np.concatenate(([0], np.cumsum([m * k for (m, _), k in zip(shapes, ks)])[:-1]))
    s_off = np.concatenate(([0], np.cumsum(ks)[:-1]))
    v_off = np.concatenate(([0], np.cumsum([k * n for (_, n), k in zip(shapes, ks)])[:-1]))
    dU, dS, dV = (backend.zeros(sum(m * k for (m, _), k in zip(shapes, ks))), backend.zeros(sum(ks)),
                  backend.zeros(sum(k * n for (_, n), k in zip(shapes, ks))))
    info, nact, transp = gpu_lib.block_svd([s[0] for s in shapes], [s[1] for s in shapes], a_off, u_off, s_off, v_off,
                                           _dev(np.concatenate([a.ravel() for a in mats])), dU, dS, dV)
    U, S, V = _host(dU), _host(dS), _host(dV)
    for a, (m, n), k, uo, so, vo, na, tr, inf in zip(mats, shapes, ks, u_off, s_off, v_off, nact, transp, info):
        u, s, vt = U[uo:uo + m * k].reshape(m, k), S[so:so + k], V[vo:vo + k * n].reshape(k, n)
        assert inf > 0
        if not a.any():
            assert na == 0, 'an all-zero block must be reported as fully deflated'
            assert np.all(s == 0.)
            side = vt @ vt.T if tr else u.T @ u        # the accumulated side; the other one is left for the caller
            assert np.max(np.abs(side - np.eye(k))) <= 4 * k * EPS
        else:
            assert na == k
            assert np.max(np.abs((u * s) @ vt - a)) <= 64 * EPS * np.linalg.norm(a)
            assert np.max(np.abs(u.T @ u - np.eye(k))) <= 64 * EPS * max(m, n)


def test_npc_svd_zero_block(gpu_lib):
    """npc.svd of an Array with a stored all-zero charge block: U and VH are isometries and U S VH = A"""
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(42)
    ci = npc.ChargeInfo([1], ['N'])
    lL = npc.LegCharge.from_qind(ci, [0, 5, 12, 20], [[0], [1], [2]], +1)
    lR = npc.LegCharge.from_qind(ci, [0, 6, 10, 13], [[0], [1], [2]], -1)
    blocks = [rng.standard_normal((5, 6)), np.zeros((7, 4)), rng.standard_normal((8, 3))]
    a = npc.Array.from_blocks([lL, lR], [[0, 0], [1, 1], [2, 2]], blocks, None, ['a', 'b'])
    U, S, VH = npc.svd(a, inner_labels=['i', 'i*'])
    u, vh, A = U.to_ndarray(), VH.to_ndarray(), a.to_ndarray()
    k = len(S)
    assert k == 5 + 4 + 3
    assert np.max(np.abs(u.T @ u - np.eye(k))) <= 64 * EPS * 20
    assert np.max(np.abs(vh @ vh.T - np.eye(k))) <= 64 * EPS * 20
    assert np.max(np.abs((u * S) @ vh - A)) <= 64 * EPS * np.linalg.norm(A)


def _eigh_inputs(rng, n):
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    w = np.repeat([-2., 0., 1., 3.5], (n + 3) // 4)[:n]                 # exact multiplicities
    yield 'multiplicities', (q * w) @ q.T
    r = max(1, n // 4)
    u, _ = np.linalg.qr(rng.standard_normal((n, r)))
    th = u * np.logspace(0, -8, r)
    yield 'low-rank psd', th @ th.T                                     # rho = theta theta^T, s in logspace(0, -8)


@pytest.fixture(params=['v3', 'v3-split', 'v1'])
def eigh_mode(request, gpu_lib):
    """pivot eigen-solver 3 (single-launch rounds while rows are <= 256 long) or with the single-launch regime off, and
    solver 1 (always three launches with column splits)"""
    old_v = gpu_lib.svd_set_eig_variant(1 if request.param == 'v1' else 3)
    old_ld = gpu_lib.svd_set_fused_max_ld(0) if request.param == 'v3-split' else None
    yield request.param
    gpu_lib.svd_set_eig_variant(old_v)
    if old_ld is not None:
        gpu_lib.svd_set_fused_max_ld(old_ld)


def _check_eigh(A, W, V, name):
    """errors in units of p eps |A|_F (eigenvalues, residual) and p eps (orthogonality), p = max(n, 16): the backward-stable
    bound with p(n) = n.  The Jacobi eigenvalue error grows ~ n: an H100 measured 0.42 .. 0.72 n eps |A|_F for the
    eigenvalues of these inputs at n = 257 .. 2048 (LAPACK as the reference)."""
    n = A.shape[0]
    p = max(n, 16)
    fro = max(np.linalg.norm(A), 1e-300)
    werr = np.max(np.abs(W - np.linalg.eigvalsh(A))) / (p * EPS * fro)
    orth = np.max(np.abs(V.T @ V - np.eye(n))) / (p * EPS)
    res = np.max(np.abs(A @ V - V * W)) / (p * EPS * fro)
    msg = '%s: eigenvalues %.3g, orthogonality %.3g, residual %.3g' % (name, werr, orth, res)
    assert werr <= 2 and orth <= 2 and res <= 2, msg                  # 2 p eps (|A|_F)


@pytest.mark.parametrize('n', [257, 600, 1024])
def test_block_eigh_large(gpu_lib, eigh_mode, n):
    """n > 256: rounds with column splits (and, for v3, single-launch rounds once few rows remain active)"""
    rng = np.random.default_rng(n)
    from tenpy_b200 import backend
    for name, A in _eigh_inputs(rng, n):
        dW, dV = backend.zeros(n), backend.zeros(n * n)
        info = gpu_lib.block_eigh([n], [0], [0], [0], _dev(A), dW, dV)
        assert info[0] > 0
        _check_eigh(A, _host(dW), _host(dV).reshape(n, n), (name, n))


def test_block_eigh_mixed_batch(gpu_lib, eigh_mode):
    """one batch of mixed sizes, laid out with gaps in NaN-filled outputs"""
    rng = np.random.default_rng(77)
    sizes = [300, 1, 40, 257, 7, 130, 2]
    mats = []
    for i, n in enumerate(sizes):
        mats.append(list(_eigh_inputs(rng, n))[i % 2])
    a_off, a_len = _layout(rng, [n * n for n in sizes])
    w_off, w_len = _layout(rng, sizes)
    v_off, v_len = _layout(rng, [n * n for n in sizes])
    Abuf = np.full(a_len, np.nan)
    for (_, A), o in zip(mats, a_off):
        Abuf[o:o + A.size] = A.ravel()
    dW, dV = _nan(w_len), _nan(v_len)
    info = gpu_lib.block_eigh(sizes, a_off, w_off, v_off, _dev(Abuf), dW, dV)
    assert np.all(info > 0)
    W, V = _host(dW), _host(dV)
    _assert_gaps_untouched(W, w_off, sizes)
    _assert_gaps_untouched(V, v_off, [n * n for n in sizes])
    for (name, A), n, wo, vo in zip(mats, sizes, w_off, v_off):
        _check_eigh(A, W[wo:wo + n], V[vo:vo + n * n].reshape(n, n), (name, n))


def test_block_eigh_2048(gpu_lib):
    """the density-matrix mixer at chi = 1024 without charges: a 2048 x 2048 low-rank PSD matrix"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(2048)
    n = 2048
    name, A = list(_eigh_inputs(rng, n))[1]
    dW, dV = backend.zeros(n), backend.zeros(n * n)
    info = gpu_lib.block_eigh([n], [0], [0], [0], _dev(A), dW, dV)
    assert info[0] > 0
    _check_eigh(A, _host(dW), _host(dV).reshape(n, n), (name, n))


# ---- int8 one-shot product ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('m,n,k,slices', [(70, 90, 150, 8), (129, 1, 17, 7), (1, 300, 65, 8), (300, 260, 500, 7)])
def test_ozaki_gemm_one_shot(gpu_lib, m, n, k, slices):
    """b200_ozaki_gemm_f64 with lda > k, ldb > n, ldc > n is bit-identical to ozaki_split + ozaki_mm, and within the
    error model of the scheme against long double; the padding columns of C stay untouched"""
    rng = np.random.default_rng(m + n + k)
    lda, ldb, ldc = k + 5, n + 3, n + 7
    A = np.full((m, lda), np.nan)
    B = np.full((k, ldb), np.nan)
    A[:, :k] = rng.standard_normal((m, k)) * np.logspace(0, -6, m)[:, None]
    B[:, :n] = rng.standard_normal((k, n)) * np.logspace(2, -3, n)[None, :]
    dA, dB = _dev(A), _dev(B)
    C1, C2 = _nan(m * ldc), _nan(m * ldc)
    gpu_lib.ozaki_gemm(m, n, k, dA, lda, dB, ldb, C1, ldc, slices)
    a_s = gpu_lib.ozaki_split(m, k, dA, lda, 1, slices)
    b_s = gpu_lib.ozaki_split(n, k, dB, 1, ldb, slices)
    gpu_lib.ozaki_mm(m, n, k, slices, a_s, b_s, C2, ldc)
    gpu_lib.ozaki_check_abort()
    c1, c2 = _host(C1).reshape(m, ldc), _host(C2).reshape(m, ldc)
    assert c1.tobytes() == c2.tobytes()
    assert np.all(np.isnan(c1[:, n:]))
    a, b = A[:, :k], B[:, :n]
    ref = a.astype(LD) @ b.astype(LD)
    den = np.abs(a) @ np.abs(b)
    bound = {7: 3e-13, 8: 3e-15}[slices]                                 # the error model of tests/test_ozaki.py
    assert np.all(np.abs(c1[:, :n] - ref) <= bound * den)
    gpu_lib.ozaki_gemm(m, n, k, dA, lda, dB, ldb, C1, ldc, slices, accumulate=True)
    gpu_lib.ozaki_mm(m, n, k, slices, a_s, b_s, C2, ldc, accumulate=True)
    assert _host(C1).tobytes() == _host(C2).tobytes()
