"""Complex decompositions: the kernels b200_block_svd_z / b200_block_qr_z against numpy on complex128 (GPU), and
npc.svd / npc.qr / npc.inner of charge-conserving ComplexArrays against dense numpy (GPU and the CPU test double of
tests/fake_device_complex.py).

Kernel checks follow tests/test_gpu_kernel_edges.py: output buffers are NaN-filled, blocks are laid out with gaps, and every
element outside the blocks must stay untouched.  Bounds (eps = 2^-52, k = min(m, n), p = max(m, n)):
* |S - S_ref| <= 32 p eps |A|_2
* |U^H U - 1|_max, |VH VH^H - 1|_max <= 32 max(k, 16) eps
* |A - U S VH|_F <= 32 p eps |A|_F
* QR: |Q^H Q - 1|_max <= 32 max(k, 16) eps, R upper triangular with a real diagonal >= 0, |QR - A|_F <= 32 p eps |A|_F
"""
import numpy as np
import pytest

EPS = np.finfo(np.float64).eps
C = 32.


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


def _crandn(rng, m, n):
    return rng.standard_normal((m, n)) + 1.j * rng.standard_normal((m, n))


def _low_rank(rng, m, n, r):
    return _crandn(rng, m, r) @ _crandn(rng, r, n)


def _degenerate(rng, m, n):
    k = min(m, n)
    u, _ = np.linalg.qr(_crandn(rng, m, k))
    v, _ = np.linalg.qr(_crandn(rng, n, k))
    s = np.repeat([3., 1., 0.5], (k + 2) // 3)[:k]          # exactly repeated singular values
    return (u * s) @ v.conj().T


def _run_svd_z(lib, rng, blocks):
    """all blocks in one call; returns per-block (U, S, VH), nact, transposed"""
    m = np.array([b.shape[0] for b in blocks], np.int64)
    n = np.array([b.shape[1] for b in blocks], np.int64)
    k = np.minimum(m, n)
    a_off, a_len = _layout(rng, m * n)
    u_off, u_len = _layout(rng, m * k)
    s_off, s_len = _layout(rng, k)
    v_off, v_len = _layout(rng, k * n)
    A = np.full(a_len, np.nan) + 1.j * np.full(a_len, np.nan)
    for o, b in zip(a_off, blocks):
        A[o:o + b.size] = b.reshape(-1)
    Ur, Ui, S, Vr, Vi = _nan(u_len), _nan(u_len), _nan(s_len), _nan(v_len), _nan(v_len)
    info, nact, transp = lib.block_svd_z(m, n, a_off, u_off, s_off, v_off, _dev(A.real), _dev(A.imag), Ur, Ui, S, Vr, Vi)
    ur, ui, s, vr, vi = (_host(t) for t in (Ur, Ui, S, Vr, Vi))
    for buf, offs, sizes in ((ur, u_off, m * k), (ui, u_off, m * k), (s, s_off, k), (vr, v_off, k * n), (vi, v_off, k * n)):
        _assert_gaps_untouched(buf, offs, sizes)
    assert np.all(info > 0)
    res = []
    for i in range(len(blocks)):
        mi, ni, ki = int(m[i]), int(n[i]), int(k[i])
        U = (ur[u_off[i]:u_off[i] + mi * ki] + 1.j * ui[u_off[i]:u_off[i] + mi * ki]).reshape(mi, ki)
        VH = (vr[v_off[i]:v_off[i] + ki * ni] + 1.j * vi[v_off[i]:v_off[i] + ki * ni]).reshape(ki, ni)
        res.append((U, s[s_off[i]:s_off[i] + ki], VH))
    return res, nact, transp


def _check_svd(A, U, S, VH, nact, transposed):
    m, n = A.shape
    k, p = min(m, n), max(m, n)
    assert np.all(np.isfinite(U)) and np.all(np.isfinite(S)) and np.all(np.isfinite(VH))
    s_ref = np.linalg.svd(A, compute_uv=False)
    n2 = s_ref[0] if k else 0.
    assert np.all(np.diff(S) <= 0.), 'S not descending'
    assert np.max(np.abs(S - s_ref)) <= C * p * EPS * n2 + 1e-300, (S[:5], s_ref[:5])
    # the deflated directions (nact..k) have a zero vector on the non-accumulated side (the caller completes it)
    r = int(nact)
    Uc, VHc = (U[:, :r], VH) if transposed else (U, VH[:r])
    ku, kv = Uc.shape[1], VHc.shape[0]
    assert np.max(np.abs(Uc.conj().T @ Uc - np.eye(ku)), initial=0.) <= C * max(k, 16) * EPS
    assert np.max(np.abs(VHc @ VHc.conj().T - np.eye(kv)), initial=0.) <= C * max(k, 16) * EPS
    if transposed:
        assert np.all(U[:, r:] == 0.)
    else:
        assert np.all(VH[r:] == 0.)
    fro = np.linalg.norm(A)
    assert np.linalg.norm(A - (U * S) @ VH) <= C * p * EPS * fro + 1e-300


SVD_SHAPES = [(1, 1), (1, 7), (9, 1), (16, 16), (17, 15), (15, 33), (32, 32), (33, 31), (40, 129), (129, 40), (128, 128),
              (127, 130), (256, 256), (257, 255), (300, 100), (64, 520)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape', SVD_SHAPES, ids=['%dx%d' % s for s in SVD_SHAPES])
def test_block_svd_z_random(gpu_lib, shape):
    rng = np.random.default_rng(sum(shape))
    A = _crandn(rng, *shape)
    (res,), nact, transp = _run_svd_z(gpu_lib, rng, [A])
    _check_svd(A, *res, nact[0], transp[0])


@pytest.mark.gpu
def test_block_svd_z_special_inputs(gpu_lib):
    """one mixed batch: zero, rank 1, rank deficient, degenerate, purely real, purely imaginary, scales 1e+-150"""
    rng = np.random.default_rng(5)
    blocks = [np.zeros((7, 5), complex), _low_rank(rng, 20, 30, 1), _low_rank(rng, 45, 40, 6), _degenerate(rng, 36, 36),
              rng.standard_normal((33, 18)) + 0.j, 1.j * rng.standard_normal((18, 50)), 1e150 * _crandn(rng, 24, 24),
              1e-150 * _crandn(rng, 19, 40), _crandn(rng, 3, 3)]
    res, nact, transp = _run_svd_z(gpu_lib, rng, blocks)
    assert nact[0] == 0 and nact[1] == 1 and nact[2] == 6
    for A, r, na, tr in zip(blocks, res, nact, transp):
        _check_svd(A, *r, na, tr)


@pytest.mark.gpu
def test_block_svd_z_2048(gpu_lib):
    rng = np.random.default_rng(2048)
    A = _crandn(rng, 2048, 2048)
    (res,), nact, transp = _run_svd_z(gpu_lib, rng, [A])
    _check_svd(A, *res, nact[0], transp[0])


def _run_qr_z(lib, rng, blocks):
    m = np.array([b.shape[0] for b in blocks], np.int64)
    n = np.array([b.shape[1] for b in blocks], np.int64)
    k = np.minimum(m, n)
    a_off, a_len = _layout(rng, m * n)
    q_off, q_len = _layout(rng, m * k)
    r_off, r_len = _layout(rng, k * n)
    A = np.full(a_len, np.nan) + 1.j * np.full(a_len, np.nan)
    for o, b in zip(a_off, blocks):
        A[o:o + b.size] = b.reshape(-1)
    Qr, Qi, Rr, Ri = _nan(q_len), _nan(q_len), _nan(r_len), _nan(r_len)
    lib.block_qr_z(m, n, a_off, q_off, r_off, _dev(A.real), _dev(A.imag), Qr, Qi, Rr, Ri)
    qr_, qi, rr, ri = (_host(t) for t in (Qr, Qi, Rr, Ri))
    for buf, offs, sizes in ((qr_, q_off, m * k), (qi, q_off, m * k), (rr, r_off, k * n), (ri, r_off, k * n)):
        _assert_gaps_untouched(buf, offs, sizes)
    out = []
    for i in range(len(blocks)):
        mi, ni, ki = int(m[i]), int(n[i]), int(k[i])
        Q = (qr_[q_off[i]:q_off[i] + mi * ki] + 1.j * qi[q_off[i]:q_off[i] + mi * ki]).reshape(mi, ki)
        R = (rr[r_off[i]:r_off[i] + ki * ni] + 1.j * ri[r_off[i]:r_off[i] + ki * ni]).reshape(ki, ni)
        out.append((Q, R))
    return out


def _check_qr(A, Q, R):
    m, n = A.shape
    k, p = min(m, n), max(m, n)
    assert np.all(np.isfinite(Q)) and np.all(np.isfinite(R))
    assert np.max(np.abs(Q.conj().T @ Q - np.eye(k))) <= C * max(k, 16) * EPS
    assert np.all(np.tril(R, -1) == 0.)
    d = np.diag(R)
    assert np.all(d.imag == 0.) and np.all(d.real >= 0.)
    assert np.linalg.norm(Q @ R - A) <= C * p * EPS * np.linalg.norm(A) + 1e-300


QR_SHAPES = [(1, 1), (1, 9), (9, 1), (16, 16), (17, 15), (33, 31), (129, 40), (40, 129), (257, 255), (400, 390), (1024, 64)]


@pytest.mark.gpu
def test_block_qr_z(gpu_lib):
    rng = np.random.default_rng(11)
    blocks = [_crandn(rng, *s) for s in QR_SHAPES]
    blocks += [np.zeros((6, 4), complex), _low_rank(rng, 30, 20, 3), rng.standard_normal((12, 9)) + 0.j,
               1.j * rng.standard_normal((9, 12)), 1e150 * _crandn(rng, 10, 10), 1e-150 * _crandn(rng, 10, 7)]
    for A, (Q, R) in zip(blocks, _run_qr_z(gpu_lib, rng, blocks)):
        _check_qr(A, Q, R)


# ---- npc level: charge-conserving ComplexArrays, CPU test double and GPU -------------------------------------------------
def _legs(npc):
    ci = npc.ChargeInfo([1], ['N'])
    lL = npc.LegCharge.from_qind(ci, [0, 5, 12, 20, 23], [[0], [1], [2], [3]], +1)
    lR = npc.LegCharge.from_qind(ci, [0, 6, 10, 13, 30], [[0], [1], [2], [4]], -1)
    return lL, lR


def _complex_array(npc, rng, kind):
    """ComplexArray with blocks (0,0) 5x6, (1,1) 7x4, (2,2) 8x3; kind 'same': both parts store all blocks,
    'differ': the parts have different block tables, 'rankdef': a rank-1 block and an all-zero block"""
    lL, lR = _legs(npc)
    qd = [[0, 0], [1, 1], [2, 2]]
    shapes = [(5, 6), (7, 4), (8, 3)]
    blocks = [_crandn(rng, *s) for s in shapes]
    if kind == 'rankdef':
        blocks[0] = _low_rank(rng, 5, 6, 1)
        blocks[1] = np.zeros((7, 4), complex)
    re = npc.Array.from_blocks([lL, lR], qd, [b.real.copy() for b in blocks], None, ['a', 'b'])
    if kind == 'differ':
        im = npc.Array.from_blocks([lL, lR], qd[1:], [b.imag.copy() for b in blocks[1:]], None, ['a', 'b'])
        blocks[0] = blocks[0].real + 0.j
    else:
        im = npc.Array.from_blocks([lL, lR], qd, [b.imag.copy() for b in blocks], None, ['a', 'b'])
    return npc.ComplexArray(re, im)


KINDS = ['same', 'differ', 'rankdef']


@pytest.fixture
def fake_device_z():
    """the numpy test double of the device library with the complex decompositions (tests/fake_device_complex.py)"""
    import fake_device_complex
    lib, restore = fake_device_complex.install()
    yield lib
    restore()


def _npc_svd_case(kind):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(KINDS.index(kind))
    a = _complex_array(npc, rng, kind)
    A = a.to_ndarray()
    U, S, VH = npc.svd(a, inner_labels=['i', 'i*'])
    assert isinstance(U, npc.ComplexArray) and isinstance(VH, npc.ComplexArray) and S.dtype == np.float64
    assert U.get_leg_labels() == ['a', 'i'] and VH.get_leg_labels() == ['i*', 'b']
    u, vh = U.to_ndarray(), VH.to_ndarray()
    kk = len(S)
    assert kk == 5 + 4 + 3
    assert np.max(np.abs(u.conj().T @ u - np.eye(kk))) <= 1e-13
    assert np.max(np.abs(vh @ vh.conj().T - np.eye(kk))) <= 1e-13
    assert np.max(np.abs((u * S) @ vh - A)) <= 1e-13 * np.linalg.norm(A)
    assert np.allclose(np.sort(S)[::-1][:np.linalg.matrix_rank(A)], np.linalg.svd(A, compute_uv=False)[:np.linalg.matrix_rank(A)],
                       rtol=0, atol=1e-13 * np.linalg.norm(A))
    # cutoff: the same legs as the real path, projected
    U2, S2, VH2 = npc.svd(a, cutoff=1e-12, inner_labels=['i', 'i*'])
    assert len(S2) == int(np.sum(S > 1e-12)) and U2.shape[1] == len(S2) and VH2.shape[0] == len(S2)
    assert np.max(np.abs((U2.to_ndarray() * S2) @ VH2.to_ndarray() - A)) <= 1e-12 * np.linalg.norm(A)
    with pytest.raises(NotImplementedError):
        npc.svd(a, guess=(U, VH))


def _npc_qr_case(kind):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(10 + KINDS.index(kind))
    a = _complex_array(npc, rng, kind)
    A = a.to_ndarray()
    Q, R = npc.qr(a, inner_labels=['q', 'q*'])
    assert isinstance(Q, npc.ComplexArray) and isinstance(R, npc.ComplexArray)
    q, r = Q.to_ndarray(), R.to_ndarray()
    assert np.max(np.abs(q.conj().T @ q - np.eye(q.shape[1]))) <= 1e-13
    assert np.max(np.abs(q @ r - A)) <= 1e-13 * np.linalg.norm(A)
    for qi in range(R.legs[0].block_number):
        blk = R.get_block([qi, qi])
        if blk is not None:
            d = np.diag(blk)
            assert np.all(np.abs(d.imag) == 0.) and np.all(d.real >= 0.)


def _npc_inner_case(kind):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(20 + KINDS.index(kind))
    a = _complex_array(npc, rng, kind)
    b = _complex_array(npc, rng, 'differ' if kind == 'same' else 'same')
    A, B = a.to_ndarray(), b.to_ndarray()
    for do_conj in (True, False):
        bb = b if do_conj else b.conj()
        ref = np.sum((A.conj() if do_conj else A) * (B if do_conj else B.conj()))
        val = npc.inner(a, bb, axes='range', do_conj=do_conj)
        assert isinstance(val, complex)
        assert abs(val - ref) <= 1e-13 * np.linalg.norm(A) * np.linalg.norm(B)
    val = npc.inner(a.re, b, axes='range', do_conj=True)            # real with complex
    assert abs(val - np.sum(A.real * B)) <= 1e-13 * np.linalg.norm(A) * np.linalg.norm(B)
    sq = a.copy()
    sq.iset_leg_labels(['a', 'b'])
    tr = npc.trace(npc.tensordot(sq, sq.conj(), axes=[[1], [1]]))
    assert isinstance(tr, complex) and abs(tr - np.linalg.norm(A)**2) <= 1e-12 * np.linalg.norm(A)**2


@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_svd_fake(fake_device_z, kind):
    _npc_svd_case(kind)


@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_qr_fake(fake_device_z, kind):
    _npc_qr_case(kind)


@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_inner_fake(fake_device_z, kind):
    _npc_inner_case(kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_svd_gpu(gpu_lib, kind):
    _npc_svd_case(kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_qr_gpu(gpu_lib, kind):
    _npc_qr_case(kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_npc_complex_inner_gpu(gpu_lib, kind):
    _npc_inner_case(kind)


def test_complex_scalar_glue(fake_device_z):
    """Array * complex -> ComplexArray (also in place and by division); expm of a ComplexArray; eigh refuses complex"""
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(3)
    lL, _ = _legs(npc)
    h = rng.standard_normal((23, 23))
    h = h + h.T
    mask = np.equal.outer(lL.to_qflat()[:, 0], lL.to_qflat()[:, 0])
    h = h * mask
    H = npc.Array.from_ndarray(h, [lL, lL.conj()], labels=['p', 'p*'])
    z = -0.05j
    for G in (H * z, z * H, H / (1. / z)):
        assert isinstance(G, npc.ComplexArray)
        assert np.max(np.abs(G.to_ndarray() - z * h)) <= 1e-15 * np.abs(h).max()
    G = H.copy()
    G *= z
    assert isinstance(G, npc.ComplexArray) and np.max(np.abs(G.to_ndarray() - z * h)) <= 1e-15 * np.abs(h).max()
    import scipy.linalg
    U = npc.expm(H * z)
    assert isinstance(U, npc.ComplexArray)
    assert np.max(np.abs(U.to_ndarray() - scipy.linalg.expm(z * h))) <= 1e-13
    with pytest.raises(NotImplementedError, match='complex Hermitian'):
        npc.eigh(H * z)
    assert npc.to_iterable_arrays('Sz') == ['Sz'] and npc.to_iterable_arrays(['Sz', ['Sx']]) == ['Sz', 'Sx']
