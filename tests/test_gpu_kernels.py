"""GPU tests of the raw C-ABI kernels against dense numpy (float64).

Tolerances: GEMM / BLAS-1 results are compared with numpy at ``1e-13 * scale`` (different summation order
in FP64); SVD / eigh are compared through gauge-invariant quantities (singular values, reconstruction,
orthonormality) like the reference's own tests (tests/test_np_conserved.py:655-720).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _dev(a):
    from tenpy_b200 import backend
    return backend.to_device(np.ascontiguousarray(a))


def test_selftest(gpu_lib):
    out = gpu_lib.selftest()
    assert out[0] < 1e-13, 'm16n8k8 DMMA fragment layout wrong: %r' % (out,)
    assert out[1] < 1e-13, 'm8n8k4 DMMA fragment layout wrong: %r' % (out,)
    assert 0 <= out[2] < 1e-11 and 0 <= out[3] < 1e-11, 'grouped gemm self test failed: %r' % (out,)


@pytest.mark.parametrize('shapes', [
    [(128, 128, 64)], [(300, 200, 100)], [(61, 33, 7), (5, 9, 122), (64, 64, 64)],
    [(1, 1, 1), (3, 1, 5), (17, 31, 2)], [(512, 384, 256), (100, 30, 7)],
    # thin products (un-bunched MPO leg: k = 1, one narrow side): streaming kernels thin_n / thin_m
    [(5000, 1, 1), (3000, 4, 2), (1, 7000, 1), (3, 2500, 3), (64, 64, 64), (8, 40, 5), (100001, 2, 1)],
    # every n, k (and k // 2 + 1) and offset even: the 16-byte (VEC) variant, at edges that are not multiples of the tile
    [(66, 34, 2), (18, 22, 10), (130, 98, 34), (6, 194, 66), (200, 130, 130)]])
def test_grouped_gemm(gpu_lib, shapes):
    from tenpy_b200 import backend
    rng = np.random.default_rng(1)
    A, B, refs = [], [], []
    m_l, n_l, c_off, pair_ptr, k_l, a_off, b_off = [], [], [], [0], [], [], []
    ao = bo = co = 0
    for (m, n, k) in shapes:
        # two products per output block, second with a different k
        acc = np.zeros((m, n))
        for kk in (k, max(1, k // 2 + 1)):
            a = rng.standard_normal((m, kk))
            b = rng.standard_normal((kk, n))
            acc += a @ b
            A.append(a.ravel())
            B.append(b.ravel())
            a_off.append(ao)
            b_off.append(bo)
            k_l.append(kk)
            ao += a.size + (-a.size) % 16
            bo += b.size + (-b.size) % 16
            A.append(np.zeros((-a.size) % 16))
            B.append(np.zeros((-b.size) % 16))
        refs.append(acc)
        m_l.append(m)
        n_l.append(n)
        c_off.append(co)
        co += m * n + (-(m * n)) % 16
        pair_ptr.append(len(k_l))
    dA, dB = _dev(np.concatenate(A)), _dev(np.concatenate(B))
    dC = backend.zeros(co)
    gpu_lib.grouped_gemm(m_l, n_l, c_off, pair_ptr, k_l, a_off, b_off, dA, dB, dC)
    C = backend.to_host(dC)
    for (m, n, k), o, ref in zip(shapes, c_off, refs):
        got = C[o:o + m * n].reshape(m, n)
        assert np.max(np.abs(got - ref)) < 1e-12 * max(1, k), (m, n, k)


def test_blas1(gpu_lib):
    from tenpy_b200 import backend
    rng = np.random.default_rng(2)
    for n in (1, 7, 1000, 2 ** 20 + 3):
        x, y = rng.standard_normal(n), rng.standard_normal(n)
        dx, dy = _dev(x), _dev(y)
        out = backend.scalar_out()
        gpu_lib.dot(n, dx, dy, backend.dot_scratch(), out)
        assert abs(backend.read_scalar(out) - np.dot(x, y)) < 1e-12 * np.sqrt(n) * 10
        gpu_lib.axpy(n, 0.37, dx, dy)
        assert np.max(np.abs(backend.to_host(dy) - (y + 0.37 * x))) < 1e-15 * 10
        gpu_lib.scal(n, -1.5, dx)
        assert np.max(np.abs(backend.to_host(dx) + 1.5 * x)) == 0.0
        w, v1, v0 = rng.standard_normal(n), rng.standard_normal(n), rng.standard_normal(n)
        dw = _dev(w)
        gpu_lib.lanczos_update(n, 0.3, _dev(v1), 0.7, _dev(v0), dw, backend.dot_scratch(), out)
        ref = w - 0.3 * v1 - 0.7 * v0
        assert np.max(np.abs(backend.to_host(dw) - ref)) < 1e-14
        assert abs(backend.read_scalar(out) - np.dot(ref, ref)) < 1e-12 * n


@pytest.mark.parametrize('shape', [(1, 1), (2, 3), (5, 5), (16, 16), (20, 10), (10, 20), (33, 47), (64, 64),
                                   (100, 37), (130, 257), (300, 300)])
def test_block_svd(gpu_lib, shape):
    from tenpy_b200 import backend
    rng = np.random.default_rng(3)
    m, n = shape
    k = min(m, n)
    A = rng.standard_normal((m, n))
    dA = _dev(A.ravel())
    dU, dS, dV = backend.zeros(m * k), backend.zeros(k), backend.zeros(k * n)
    info, nact, _ = gpu_lib.block_svd([m], [n], [0], [0], [0], [0], dA, dU, dS, dV)
    assert nact[0] == k
    U = backend.to_host(dU).reshape(m, k)
    S = backend.to_host(dS)
    VT = backend.to_host(dV).reshape(k, n)
    Sref = np.linalg.svd(A, compute_uv=False)
    assert info[0] > 0
    assert np.all(np.diff(S) <= 1e-14)
    assert np.max(np.abs(S - Sref)) < 1e-12 * Sref[0]
    assert np.max(np.abs(U @ np.diag(S) @ VT - A)) < 1e-12 * Sref[0]
    assert np.max(np.abs(U.T @ U - np.eye(k))) < 1e-12
    assert np.max(np.abs(VT @ VT.T - np.eye(k))) < 1e-12
    assert np.max(np.abs(backend.to_host(dA).reshape(m, n) - A)) == 0.0  # input untouched


@pytest.fixture(params=[1, 3])
def eig_variant(request, gpu_lib):
    """both pivot eigen-solvers of the Jacobi rounds (csrc/svd.cu: 1 = shared memory, 3 = registers + shuffles)"""
    old = gpu_lib.svd_set_eig_variant(request.param)
    yield request.param
    gpu_lib.svd_set_eig_variant(old)


@pytest.mark.parametrize('shape', [(5, 5), (33, 47), (64, 64), (200, 150), (300, 512)])
def test_block_svd_eig_variants(gpu_lib, eig_variant, shape):
    """the block SVD with either pivot eigen-solver: singular values, reconstruction, orthogonality against LAPACK"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(11)
    m, n = shape
    k = min(m, n)
    A = rng.standard_normal((m, n)) * np.logspace(0, -5, n)[None, :]
    dA = _dev(A.ravel())
    dU, dS, dV = backend.zeros(m * k), backend.zeros(k), backend.zeros(k * n)
    info, nact, _ = gpu_lib.block_svd([m], [n], [0], [0], [0], [0], dA, dU, dS, dV)
    U, S, VT = backend.to_host(dU).reshape(m, k), backend.to_host(dS), backend.to_host(dV).reshape(k, n)
    Sref = np.linalg.svd(A, compute_uv=False)
    assert info[0] > 0 and nact[0] == k
    assert np.max(np.abs(S - Sref)) < 1e-12 * Sref[0]
    assert np.max(np.abs(U @ np.diag(S) @ VT - A)) < 1e-12 * Sref[0]
    assert np.max(np.abs(U.T @ U - np.eye(k))) < 1e-12
    assert np.max(np.abs(VT @ VT.T - np.eye(k))) < 1e-12


@pytest.mark.parametrize('inner', [2, 1, 0])
@pytest.mark.parametrize('fused_ld', [0, 512])
def test_block_svd_round_regimes(gpu_lib, inner, fused_ld):
    """the two regimes of a Jacobi round -- three launches with column splits / one launch per round (small blocks) -- and the
    modes of the pivot eigen-solver (2 or 1 inner sweeps, cross mode = 0) on a batch that mixes both block sizes"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(21)
    shapes = [(300, 260), (130, 400), (48, 48), (17, 5), (96, 31)]
    mats = [rng.standard_normal(sh) * np.logspace(0, -6, sh[1])[None, :] for sh in shapes]
    a_off, u_off, s_off, v_off = [], [], [], []
    ao = uo = so = vo = 0
    for (m, n) in shapes:
        k = min(m, n)
        a_off.append(ao), u_off.append(uo), s_off.append(so), v_off.append(vo)
        ao, uo, so, vo = ao + m * n, uo + m * k, so + k, vo + k * n
    dA = _dev(np.concatenate([a.ravel() for a in mats]))
    dU, dS, dV = backend.zeros(uo), backend.zeros(so), backend.zeros(vo)
    old_in, old_ld = gpu_lib.svd_set_eig_inner_sweeps(inner), gpu_lib.svd_set_fused_max_ld(fused_ld)
    try:
        info, nact, _ = gpu_lib.block_svd([s[0] for s in shapes], [s[1] for s in shapes], a_off, u_off, s_off, v_off, dA, dU, dS, dV)
    finally:
        gpu_lib.svd_set_eig_inner_sweeps(old_in)
        gpu_lib.svd_set_fused_max_ld(old_ld)
    U, S, V = backend.to_host(dU), backend.to_host(dS), backend.to_host(dV)
    for (m, n), A, u, s_, v, na in zip(shapes, mats, u_off, s_off, v_off, nact):
        k = min(m, n)
        Ui, Si, Vi = U[u:u + m * k].reshape(m, k), S[s_:s_ + k], V[v:v + k * n].reshape(k, n)
        Sref = np.linalg.svd(A, compute_uv=False)
        assert na == k
        assert np.max(np.abs(Si - Sref)) < 1e-12 * Sref[0]
        assert np.max(np.abs(Ui @ np.diag(Si) @ Vi - A)) < 1e-12 * Sref[0]
        assert np.max(np.abs(Ui.T @ Ui - np.eye(k))) < 1e-12
        assert np.max(np.abs(Vi @ Vi.T - np.eye(k))) < 1e-12


def test_block_svd_4096_rows_active_set(gpu_lib):
    """q = 4096 vectors (the two-site wave function at chi = 2048): the device-side active-set bookkeeping sorts 4096 row
    norms in shared memory (48 KB + the kernel's static shared memory: opt-in limit); numerically low-rank input"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(8)
    n, r = 4096, 40
    q1, _ = np.linalg.qr(rng.standard_normal((n, r)))
    q2, _ = np.linalg.qr(rng.standard_normal((n, r)))
    sv = np.logspace(0, -6, r)
    A = (q1 * sv) @ q2.T
    dA = _dev(A.ravel())
    dU, dS, dV = backend.zeros(n * n), backend.zeros(n), backend.zeros(n * n)
    old = gpu_lib.svd_set_deflation_tol(1e-10)
    try:
        info, nact, _ = gpu_lib.block_svd([n], [n], [0], [0], [0], [0], dA, dU, dS, dV)
    finally:
        gpu_lib.svd_set_deflation_tol(old)
    S = backend.to_host(dS)
    assert info[0] > 0 and r <= nact[0] < 200
    assert np.max(np.abs(S[:r] - sv)) < 1e-11       # (measured 1.1e-12: directions below 1e-10 |A| are deflated, not iterated)
    U = backend.to_host(dU).reshape(n, n)[:, :r]
    VT = backend.to_host(dV).reshape(n, n)[:r]
    assert np.max(np.abs((U * S[:r]) @ VT - A)) < 1e-9
    assert np.max(np.abs(U.T @ U - np.eye(r))) < 1e-12


def test_block_svd_batch_graded(gpu_lib):
    """several blocks of different shapes in one batch, with strongly graded singular values"""
    from tenpy_b200 import backend
    rng = np.random.default_rng(4)
    shapes = [(40, 40), (7, 8), (122, 119), (64, 20), (3, 90)]
    mats, a_off, u_off, s_off, v_off = [], [], [], [], []
    ao = uo = so = vo = 0
    for (m, n) in shapes:
        k = min(m, n)
        q1, _ = np.linalg.qr(rng.standard_normal((m, k)))
        q2, _ = np.linalg.qr(rng.standard_normal((n, k)))
        s = np.logspace(0, -12, k)
        mats.append((q1 * s) @ q2.T)
        a_off.append(ao), u_off.append(uo), s_off.append(so), v_off.append(vo)
        ao += m * n
        uo += m * k
        so += k
        vo += k * n
    dA = _dev(np.concatenate([a.ravel() for a in mats]))
    dU, dS, dV = backend.zeros(uo), backend.zeros(so), backend.zeros(vo)
    gpu_lib.block_svd([s[0] for s in shapes], [s[1] for s in shapes], a_off, u_off, s_off, v_off, dA, dU, dS, dV)
    U, S, V = backend.to_host(dU), backend.to_host(dS), backend.to_host(dV)
    for (m, n), A, a, u, s, v in zip(shapes, mats, a_off, u_off, s_off, v_off):
        k = min(m, n)
        Ui, Si, Vi = U[u:u + m * k].reshape(m, k), S[s:s + k], V[v:v + k * n].reshape(k, n)
        Sref = np.linalg.svd(A, compute_uv=False)
        assert np.max(np.abs(Si - Sref)) < 1e-13
        assert np.max(np.abs(Ui @ np.diag(Si) @ Vi - A)) < 1e-13
        big = Si > 1e-9
        assert np.max(np.abs(Ui[:, big].T @ Ui[:, big] - np.eye(big.sum()))) < 1e-10
        assert np.max(np.abs(Vi[big] @ Vi[big].T - np.eye(big.sum()))) < 1e-10


@pytest.mark.parametrize('n', [1, 2, 7, 16, 33, 64, 150])
def test_block_eigh(gpu_lib, n):
    from tenpy_b200 import backend
    rng = np.random.default_rng(5)
    X = rng.standard_normal((n, n))
    for A in (X + X.T, X @ X.T / n):
        dA = _dev(A.ravel())
        dW, dV = backend.zeros(n), backend.zeros(n * n)
        gpu_lib.block_eigh([n], [0], [0], [0], dA, dW, dV)
        W, V = backend.to_host(dW), backend.to_host(dV).reshape(n, n)
        Wref = np.linalg.eigvalsh(A)
        scale = max(1.0, np.abs(Wref).max())
        assert np.max(np.abs(W - Wref)) < 1e-12 * scale
        assert np.max(np.abs(V @ np.diag(W) @ V.T - A)) < 1e-11 * scale
        assert np.max(np.abs(V.T @ V - np.eye(n))) < 1e-12
