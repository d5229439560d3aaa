"""GPU tests of the block decompositions across the whole double range: exact power-of-two equivariance.

Multiplying a matrix by 2^e is exact, and it commutes with every floating-point operation in the normal range.  So a
correct kernel, given 2^e A, returns the same U, VT, Q and V bit for bit, S, R and W multiplied by exactly 2^e, and the
same info / nact / transposed -- for every e that keeps the inputs normal.  The base blocks have entries with magnitudes
in [2^-30, 2^4], so 2^e A is normal for |e| <= 990; together with the accuracy checks at e = 0 (here and in
test_gpu_kernel_edges.py) this gives the accuracy of every kernel across the range, with no tolerance to tune.

Each kernel first has to be deterministic: one batch is run twice and must agree bit for bit.  Every batch mixes the same
base blocks at all scales (2^-990 next to 2^+990), laid out with gaps in NaN-filled outputs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
EXPS = [-990, -700, -540, -300, -270, -260, -80, 0, 80, 260, 270, 300, 540, 700, 990]


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


def _bounded(rng, shape):
    """Gaussian entries with magnitudes clamped to [2^-30, 15]"""
    x = rng.standard_normal(shape)
    return np.copysign(np.clip(np.abs(x), 2.**-30, 15.), x)


def _complexify(rng, bases):
    """complex counterparts: a random bounded imaginary part where the real part is nonzero, (1 + 2i) A for the
    rank-deficient blocks (the same rank)"""
    return [(nm, A * (1 + 2j) if nm.startswith('rankdef') else A + 1j * _bounded(rng, A.shape) * (A != 0))
            for nm, A in bases]


def _int_low_rank(rng, m, n, r):
    """exactly rank r, small integer entries (exact zeros possible)"""
    return (rng.integers(-3, 4, (m, r)) @ rng.integers(-3, 4, (r, n))).astype(np.float64)


def _svd_bases(rng, big):
    """tall, wide, square, rank-deficient and zero blocks; `big` adds a block with rows longer than 256 (three-launch
    rounds with column splits, the fused regime ends at 256)"""
    b = [('tall', _bounded(rng, (40, 25))), ('wide', _bounded(rng, (25, 40))), ('square', _bounded(rng, (33, 33))),
         ('rankdef', _int_low_rank(rng, 30, 30, 5)), ('rankdef-tall', _int_low_rank(rng, 50, 20, 3)),
         ('zero', np.zeros((6, 4)))]
    if big:
        b.append(('split', _bounded(rng, (300, 270))))
    return b


@pytest.fixture(params=['v3', 'v3-split', 'v1', 'cross'])
def solver(request, gpu_lib):
    """pivot eigen-solver 3 (fused single-launch rounds while rows are <= 256 long), 3 with the fused regime off,
    solver 1 (three launches), and the cross mode of solver 3 (svd_set_eig_inner_sweeps(0))"""
    old_v = gpu_lib.svd_set_eig_variant(1 if request.param == 'v1' else 3)
    old_ld = gpu_lib.svd_set_fused_max_ld(0) if request.param == 'v3-split' else None
    old_in = gpu_lib.svd_set_eig_inner_sweeps(0) if request.param == 'cross' else None
    yield request.param
    gpu_lib.svd_set_eig_variant(old_v)
    if old_ld is not None:
        gpu_lib.svd_set_fused_max_ld(old_ld)
    if old_in is not None:
        gpu_lib.svd_set_eig_inner_sweeps(old_in)


def _ldexp(A, e):
    """2^e A, also for complex A (exact for the inputs here)"""
    if np.iscomplexobj(A):
        out = np.empty(A.shape, complex)
        out.real, out.imag = np.ldexp(A.real, e), np.ldexp(A.imag, e)
        return out
    return np.ldexp(A, e)


def _scaled_batch(bases, exps):
    """every base block at every exponent: list of (base index, e, 2^e A)"""
    return [(i, e, _ldexp(A, e)) for i, (_, A) in enumerate(bases) for e in exps]


# ---- SVD ------------------------------------------------------------------------------------------------------------------

def _run_svd(lib, rng, mats, cplx):
    shapes = [A.shape for A in mats]
    ks = [min(s) for s in shapes]
    a_off, a_len = _layout(rng, [m * n for m, n in shapes])
    u_off, u_len = _layout(rng, [m * k for (m, _), k in zip(shapes, ks)])
    s_off, s_len = _layout(rng, ks)
    v_off, v_len = _layout(rng, [k * n for (_, n), k in zip(shapes, ks)])
    planes = 2 if cplx else 1
    A_h = [np.full(a_len, np.nan) for _ in range(planes)]
    for A, o in zip(mats, a_off):
        A_h[0][o:o + A.size] = A.real.ravel()
        if cplx:
            A_h[1][o:o + A.size] = A.imag.ravel()
    dA = [_dev(x) for x in A_h]
    dU, dV = [_nan(u_len) for _ in range(planes)], [_nan(v_len) for _ in range(planes)]
    dS = _nan(s_len)
    if cplx:
        info, nact, tr = lib.block_svd_z([s[0] for s in shapes], [s[1] for s in shapes], a_off, u_off, s_off, v_off,
                                         dA[0], dA[1], dU[0], dU[1], dS, dV[0], dV[1])
    else:
        info, nact, tr = lib.block_svd([s[0] for s in shapes], [s[1] for s in shapes], a_off, u_off, s_off, v_off,
                                       dA[0], dU[0], dS, dV[0])
    U = [_host(x) for x in dU]
    V = [_host(x) for x in dV]
    S = _host(dS)
    _assert_gaps_untouched(S, s_off, ks)
    for x in U:
        _assert_gaps_untouched(x, u_off, [m * k for (m, _), k in zip(shapes, ks)])
    for x in V:
        _assert_gaps_untouched(x, v_off, [k * n for (_, n), k in zip(shapes, ks)])
    out = []
    for i, ((m, n), k) in enumerate(zip(shapes, ks)):
        u = sum(x[u_off[i]:u_off[i] + m * k] * f for x, f in zip(U, (1, 1j))).reshape(m, k)
        vt = sum(x[v_off[i]:v_off[i] + k * n] * f for x, f in zip(V, (1, 1j))).reshape(k, n)
        out.append((u, S[s_off[i]:s_off[i] + k], vt, int(info[i]), int(nact[i]), int(tr[i])))
    return out


def _same_bits(x, y):
    return x.shape == y.shape and np.array_equal(x, y)      # NaN anywhere fails


def _check_equivariant(batch, res, nvec, nval, what):
    """res[j] = (vectors..., values, ints...) of batch[j] = (base, e, 2^e A): vectors equal to those at e = 0 bit for bit,
    values equal to 2^e times those at e = 0 exactly, the integers equal"""
    ref = {i: r for (i, e, _), r in zip(batch, res) if e == 0}
    bad = []
    for (i, e, _), r in zip(batch, res):
        r0 = ref[i]
        ok = all(_same_bits(np.asarray(r[t]), np.asarray(r0[t])) for t in nvec)
        ok = ok and all(_same_bits(np.asarray(r[t]), np.ldexp(np.asarray(r0[t]), e)) for t in nval)
        ok = ok and all(r[t] == r0[t] for t in range(len(r)) if t not in nvec and t not in nval)
        if not ok:
            bad.append((i, e))
    assert not bad, '%s: not equivariant for (base, e) = %s' % (what, bad)


def _check_svd_accuracy(A, u, s, vt, nact, transposed):
    """e = 0: S against LAPACK to 8 max(m, n) eps |A|_F; U S VT = A to 8 max(m, n) eps |A|_F; the accumulated side
    orthonormal to 8 max(m, n) eps (the other side is zero for the nact.. directions, filled by npc.svd)"""
    m, n = A.shape
    k = min(m, n)
    fro = np.linalg.norm(A)
    tol = 8 * max(m, n) * EPS
    assert np.max(np.abs(s - np.linalg.svd(A, compute_uv=False)), initial=0.) <= tol * fro
    assert np.max(np.abs((u * s) @ vt - A), initial=0.) <= tol * max(fro, 1e-300) or fro == 0.
    acc = vt if transposed else u.conj().T
    assert np.max(np.abs(acc @ acc.conj().T - np.eye(k))) <= tol
    assert 0 <= nact <= k


@pytest.mark.parametrize('big', [False, True], ids=['fused-sizes', 'split-sizes'])
def test_block_svd_scale_equivariance(gpu_lib, solver, big):
    rng = np.random.default_rng(1 + big)
    bases = _svd_bases(rng, big)
    exps = EXPS if not big else [-990, -540, -270, 0, 260, 540, 990]
    batch = _scaled_batch(bases, exps)
    mats = [A for _, _, A in batch]
    res = _run_svd(gpu_lib, np.random.default_rng(3), mats, False)
    again = _run_svd(gpu_lib, np.random.default_rng(3), mats, False)
    for r, r2 in zip(res, again):                  # deterministic from run to run
        assert all(_same_bits(np.asarray(x), np.asarray(y)) for x, y in zip(r, r2))
    for (i, e, A), (u, s, vt, info, nact, tr) in zip(batch, res):
        assert info > 0
        if e == 0:
            _check_svd_accuracy(A, u, s, vt, nact, tr)
        if e == 990:
            assert np.isfinite(s[0]) and np.isfinite(np.linalg.norm(A / 2.**990) * 2.**990)
    _check_equivariant(batch, res, nvec=(0, 2), nval=(1,), what='block_svd[%s]' % solver)


def test_block_svd_z_scale_equivariance(gpu_lib):
    rng = np.random.default_rng(4)
    bases = _complexify(rng, _svd_bases(rng, True))
    batch = _scaled_batch(bases, EXPS)
    mats = [A for _, _, A in batch]
    res = _run_svd(gpu_lib, np.random.default_rng(5), mats, True)
    again = _run_svd(gpu_lib, np.random.default_rng(5), mats, True)
    for r, r2 in zip(res, again):
        assert all(_same_bits(np.asarray(x), np.asarray(y)) for x, y in zip(r, r2))
    for (i, e, A), (u, s, vt, info, nact, tr) in zip(batch, res):
        assert info > 0
        if e == 0:
            _check_svd_accuracy(A, u, s, vt, nact, tr)
    _check_equivariant(batch, res, nvec=(0, 2), nval=(1,), what='block_svd_z')


def test_block_svd_subnormal_entries(gpu_lib, solver):
    """blocks of subnormal entries (A' 2^-1060, rounded on input): checked against LAPACK on the exactly rescaled input
    A'' = 2^1060 A (scaling subnormals up is exact).  S is subnormal on output, rounded once: its bound has the absolute
    term 2^-1074 (2^-14 after rescaling)."""
    rng = np.random.default_rng(6)
    mats = [np.ldexp(_bounded(rng, s), -1060) for s in [(12, 9), (9, 12), (20, 20)]]
    res = _run_svd(gpu_lib, rng, mats, False)
    for A, (u, s, vt, info, nact, tr) in zip(mats, res):
        A2 = np.ldexp(A, 1060)
        m, n = A.shape
        fro = np.linalg.norm(A2)
        s2 = np.linalg.svd(A2, compute_uv=False)
        assert info > 0 and nact == min(m, n)
        # 8 max(m, n) eps |A''|_F, plus one rounding of a subnormal S
        assert np.max(np.abs(np.ldexp(s, 1060) - s2)) <= 8 * max(m, n) * EPS * fro + 2.**-14
        assert np.max(np.abs(u.T @ u - np.eye(min(m, n)))) <= 8 * max(m, n) * EPS
        assert np.max(np.abs(vt @ vt.T - np.eye(min(m, n)))) <= 8 * max(m, n) * EPS
        # the vectors diagonalise A'': U^T A'' V = diag(S'') to 8 max(m, n) eps |A''|_F
        assert np.max(np.abs(u.T @ A2 @ vt.T - np.diag(s2))) <= 8 * max(m, n) * EPS * fro


def test_block_svd_graded_no_deflation(gpu_lib, solver):
    """row-graded blocks A = diag(d) Q (Q with orthonormal rows) whose singular values d span 1 .. 1e-250 within one
    block, with deflation off: the configuration of the retry after B200_ERR_NOCONV.  Rows below ~1e-154 have Gram
    products (and, below ~1e-162, squared norms) that underflow.  The block must converge at the first attempt, S must be
    within 8 max(m, n) eps S_max of LAPACK, and U and VT must be orthonormal to 8 max(m, n) eps."""
    rng = np.random.default_rng(21)
    mats = []
    for m, n in [(40, 40), (24, 40)]:
        q = np.linalg.qr(rng.standard_normal((n, m)))[0].T
        mats.append(np.logspace(0, -250, m)[:, None] * q)
    old = gpu_lib.svd_set_deflation(False)
    retries = gpu_lib.noconv_retries
    try:
        res = _run_svd(gpu_lib, np.random.default_rng(22), mats, False)
    finally:
        gpu_lib.svd_set_deflation(old)
    assert gpu_lib.noconv_retries == retries, 'needed the retry after B200_ERR_NOCONV'
    for A, (u, s, vt, info, nact, tr) in zip(mats, res):
        m, n = A.shape
        k = min(m, n)
        tol = 8 * max(m, n) * EPS
        s_ref = np.linalg.svd(A, compute_uv=False)
        assert info > 0 and nact == k
        assert np.max(np.abs(s - s_ref)) <= tol * s_ref[0], (s, s_ref)
        assert np.max(np.abs(u.T @ u - np.eye(k))) <= tol
        assert np.max(np.abs(vt @ vt.T - np.eye(k))) <= tol


# ---- eigh -----------------------------------------------------------------------------------------------------------------

def _run_eigh(lib, rng, mats):
    sizes = [A.shape[0] for A in mats]
    a_off, a_len = _layout(rng, [n * n for n in sizes])
    w_off, w_len = _layout(rng, sizes)
    v_off, v_len = _layout(rng, [n * n for n in sizes])
    Abuf = np.full(a_len, np.nan)
    for A, o in zip(mats, a_off):
        Abuf[o:o + A.size] = A.ravel()
    dW, dV = _nan(w_len), _nan(v_len)
    info = lib.block_eigh(sizes, a_off, w_off, v_off, _dev(Abuf), dW, dV)
    W, V = _host(dW), _host(dV)
    _assert_gaps_untouched(W, w_off, sizes)
    _assert_gaps_untouched(V, v_off, [n * n for n in sizes])
    return [(V[v_off[i]:v_off[i] + n * n].reshape(n, n), W[w_off[i]:w_off[i] + n], int(info[i]))
            for i, n in enumerate(sizes)]


@pytest.mark.parametrize('big', [False, True], ids=['fused-sizes', 'split-sizes'])
def test_block_eigh_scale_equivariance(gpu_lib, solver, big):
    rng = np.random.default_rng(7 + big)
    bases = []
    for n in ([1, 7, 40, 130] if not big else [300]):
        x = np.triu(_bounded(rng, (n, n)))
        bases.append(('sym%d' % n, x + np.triu(x, 1).T))
    r = _int_low_rank(rng, 24, 3, 3)
    bases.append(('psd-rankdef', r @ r.T))
    bases.append(('zero', np.zeros((5, 5))))
    exps = EXPS if not big else [-990, -540, -270, 0, 260, 540, 990]
    batch = _scaled_batch(bases, exps)
    mats = [A for _, _, A in batch]
    res = _run_eigh(gpu_lib, np.random.default_rng(9), mats)
    again = _run_eigh(gpu_lib, np.random.default_rng(9), mats)
    for r1, r2 in zip(res, again):
        assert all(_same_bits(np.asarray(x), np.asarray(y)) for x, y in zip(r1, r2))
    for (i, e, A), (V, W, info) in zip(batch, res):
        assert info > 0
        if e == 0:
            n = A.shape[0]
            p = max(n, 16)
            fro = max(np.linalg.norm(A), 1e-300)
            # test_gpu_kernel_edges._check_eigh: 2 p eps |A|_F, p = max(n, 16); orthogonality 2 p eps
            assert np.max(np.abs(W - np.linalg.eigvalsh(A))) <= 2 * p * EPS * fro
            assert np.max(np.abs(V.T @ V - np.eye(n))) <= 2 * p * EPS
            assert np.max(np.abs(A @ V - V * W)) <= 2 * p * EPS * fro
    _check_equivariant(batch, res, nvec=(0,), nval=(1,), what='block_eigh[%s]' % solver)


# ---- QR -------------------------------------------------------------------------------------------------------------------

def _run_qr(lib, rng, mats, cplx):
    shapes = [A.shape for A in mats]
    ks = [min(s) for s in shapes]
    a_off, a_len = _layout(rng, [m * n for m, n in shapes])
    q_off, q_len = _layout(rng, [m * k for (m, _), k in zip(shapes, ks)])
    r_off, r_len = _layout(rng, [k * n for (_, n), k in zip(shapes, ks)])
    planes = 2 if cplx else 1
    A_h = [np.full(a_len, np.nan) for _ in range(planes)]
    for A, o in zip(mats, a_off):
        A_h[0][o:o + A.size] = A.real.ravel()
        if cplx:
            A_h[1][o:o + A.size] = A.imag.ravel()
    dA = [_dev(x) for x in A_h]
    dQ, dR = [_nan(q_len) for _ in range(planes)], [_nan(r_len) for _ in range(planes)]
    ms, ns = [s[0] for s in shapes], [s[1] for s in shapes]
    if cplx:
        lib.block_qr_z(ms, ns, a_off, q_off, r_off, dA[0], dA[1], dQ[0], dQ[1], dR[0], dR[1])
    else:
        lib.block_qr(ms, ns, a_off, q_off, r_off, dA[0], dQ[0], dR[0])
    Q, R = [_host(x) for x in dQ], [_host(x) for x in dR]
    for x in Q:
        _assert_gaps_untouched(x, q_off, [m * k for (m, _), k in zip(shapes, ks)])
    for x in R:
        _assert_gaps_untouched(x, r_off, [k * n for (_, n), k in zip(shapes, ks)])
    out = []
    for i, ((m, n), k) in enumerate(zip(shapes, ks)):
        out.append((tuple(x[q_off[i]:q_off[i] + m * k].reshape(m, k) for x in Q),
                    tuple(x[r_off[i]:r_off[i] + k * n].reshape(k, n) for x in R)))
    return out


@pytest.mark.parametrize('cplx', [False, True], ids=['real', 'complex'])
def test_block_qr_scale_equivariance(gpu_lib, cplx):
    rng = np.random.default_rng(10 + cplx)
    bases = [('tall', _bounded(rng, (40, 25))), ('wide', _bounded(rng, (25, 40))), ('square', _bounded(rng, (33, 33))),
             ('rankdef', _int_low_rank(rng, 30, 30, 5)), ('zero', np.zeros((6, 4))), ('long', _bounded(rng, (300, 20)))]
    if cplx:
        bases = _complexify(rng, bases)
    batch = _scaled_batch(bases, EXPS)
    mats = [A for _, _, A in batch]
    res = _run_qr(gpu_lib, np.random.default_rng(12), mats, cplx)
    again = _run_qr(gpu_lib, np.random.default_rng(12), mats, cplx)
    for r1, r2 in zip(res, again):
        assert all(_same_bits(x, y) for t in range(2) for x, y in zip(r1[t], r2[t]))
    for (i, e, A), (Q, R) in zip(batch, res):
        if e == 0:
            q = Q[0] + (1j * Q[1] if cplx else 0)
            r = R[0] + (1j * R[1] if cplx else 0)
            m, n = A.shape
            # |QR - A| <= 8 max(m, n) eps |A|_F, |Q^H Q - 1| <= 8 max(m, n) eps
            assert np.max(np.abs(q @ r - A)) <= 8 * max(m, n) * EPS * np.linalg.norm(A)
            assert np.max(np.abs(q.conj().T @ q - np.eye(min(m, n)))) <= 8 * max(m, n) * EPS
    flat = [Q + R for Q, R in res]       # (Q planes..., R planes...)
    planes = 2 if cplx else 1
    _check_equivariant(batch, flat, nvec=tuple(range(planes)), nval=tuple(range(planes, 2 * planes)),
                       what='block_qr%s' % ('_z' if cplx else ''))
