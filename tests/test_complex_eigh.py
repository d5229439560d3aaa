"""Complex Hermitian eigen-decomposition: the kernel b200_block_eigh_z against numpy.linalg.eigh on dense complex
Hermitian blocks (GPU), and npc.eigh / npc.eigvalsh of charge-conserving ComplexArrays against dense numpy (GPU and the
CPU test double of tests/fake_device_eigh_z.py).

Kernel bounds, in the units of test_gpu_kernel_edges._check_eigh (p = max(n, 16), eps = 2^-52):
* eigenvalues |W - W_ref|_max and residual |A V - V W|_max <= 4 p eps |A|_F
* orthogonality |V^H V - 1|_max <= 4 p eps
An H100 80GB HBM3 (700 W power limit) measured at most 0.87 (eigenvalues, low-rank PSD), 0.97 (orthogonality,
multiplicities) and 0.36 (residual) of these units over the inputs of test_block_eigh_z_kernel; complex eigenvalues of a
real symmetric block lay within 0.55 p eps |A|_F of the real kernel's (bound: 4).
"""
import numpy as np
import pytest

EPS = np.finfo(np.float64).eps
C = 4.
KERNEL_SIZES = [1, 2, 15, 16, 17, 31, 32, 33, 100, 256, 257, 600, 1024]


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


def _unitary(rng, n):
    q, r = np.linalg.qr(_crandn(rng, n, n))
    return q


def _hermitian_inputs(rng, n):
    """(name, A): Q diag(w) Q^H with exact multiplicities, low-rank PSD, real symmetric (Im = 0), i times a real
    antisymmetric matrix (Re = 0), zero"""
    q = _unitary(rng, n)
    w = rng.choice([-2., -0.5, 0., 1., 3.], n)
    yield 'multiplicities', (q * w) @ q.conj().T
    r = max(1, n // 3)
    theta = q[:, :r] * np.logspace(0, -8, r)
    yield 'psd-lowrank', theta @ theta.conj().T
    x = rng.standard_normal((n, n))
    yield 'real', (x + x.T) + 0.j
    yield 'imag', 1.j * (x - x.T)
    yield 'zero', np.zeros((n, n), dtype=np.complex128)


def _run_eigh_z(lib, rng, mats):
    """one b200_block_eigh_z batch over `mats`, laid out with gaps in NaN-filled outputs; [(W, V, info)]"""
    sizes = [A.shape[0] for A in mats]
    a_off, a_len = _layout(rng, [n * n for n in sizes])
    w_off, w_len = _layout(rng, sizes)
    v_off, v_len = _layout(rng, [n * n for n in sizes])
    Are, Aim = np.full(a_len, np.nan), np.full(a_len, np.nan)
    for A, o in zip(mats, a_off):
        Are[o:o + A.size] = A.real.ravel()
        Aim[o:o + A.size] = A.imag.ravel()
    dW, dVr, dVi = _nan(w_len), _nan(v_len), _nan(v_len)
    info = lib.block_eigh_z(sizes, a_off, w_off, v_off, _dev(Are), _dev(Aim), dW, dVr, dVi)
    W, Vr, Vi = _host(dW), _host(dVr), _host(dVi)
    _assert_gaps_untouched(W, w_off, sizes)
    for V in (Vr, Vi):
        _assert_gaps_untouched(V, v_off, [n * n for n in sizes])
    return [(W[w_off[i]:w_off[i] + n], Vr[v_off[i]:v_off[i] + n * n].reshape(n, n),
             Vi[v_off[i]:v_off[i] + n * n].reshape(n, n), int(info[i])) for i, n in enumerate(sizes)]


def _errors(A, W, V):
    n = A.shape[0]
    p = max(n, 16)
    fro = max(np.linalg.norm(A), 1e-300)
    werr = np.max(np.abs(W - np.linalg.eigvalsh(A))) / (p * EPS * fro)
    orth = np.max(np.abs(V.conj().T @ V - np.eye(n))) / (p * EPS)
    res = np.max(np.abs(A @ V - V * W)) / (p * EPS * fro)
    return werr, orth, res


def _check(A, W, V, name):
    werr, orth, res = _errors(A, W, V)
    assert np.all(np.diff(W) >= 0.), (name, 'W not ascending')
    assert werr <= C and orth <= C and res <= C, '%s: eigenvalues %.3g, orthogonality %.3g, residual %.3g' % (
        name, werr, orth, res)


# ---- kernel ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('n', KERNEL_SIZES)
def test_block_eigh_z_kernel(gpu_lib, n):
    from tenpy_b200 import backend
    rng = np.random.default_rng(1000 + n)
    for name, A in _hermitian_inputs(rng, n):
        (W, Vr, Vi, info), = _run_eigh_z(gpu_lib, rng, [A])
        assert info > 0, (name, n)
        _check(A, W, Vr + 1.j * Vi, (name, n))
        if name == 'real':      # the real kernel on the same matrix: the same eigenvalues within rounding
            dW, dV = backend.zeros(n), backend.zeros(n * n)
            gpu_lib.block_eigh([n], [0], [0], [0], _dev(A.real), dW, dV)
            p = max(n, 16)
            assert np.max(np.abs(W - _host(dW))) <= C * p * EPS * np.linalg.norm(A), n


@pytest.mark.gpu
def test_block_eigh_z_mixed_batch(gpu_lib):
    """one batch of several sizes and every kind of input"""
    rng = np.random.default_rng(77)
    sizes = [300, 1, 40, 257, 7, 130, 2, 33]
    mats, names = [], []
    for i, n in enumerate(sizes):
        name, A = list(_hermitian_inputs(rng, n))[i % 5]
        mats.append(A)
        names.append(name)
    for A, name, (W, Vr, Vi, info) in zip(mats, names, _run_eigh_z(gpu_lib, rng, mats)):
        assert info > 0
        _check(A, W, Vr + 1.j * Vi, (name, A.shape[0]))


@pytest.mark.gpu
@pytest.mark.parametrize('big', [False, True], ids=['fused-sizes', 'split-sizes'])
def test_block_eigh_z_scale_equivariance(gpu_lib, big):
    """a block times 2^e: V bit for bit that of the block, W exactly 2^e times its W (as the real eigh in
    test_gpu_scale_range.py)"""
    from test_gpu_scale_range import EXPS, _bounded, _check_equivariant, _scaled_batch
    rng = np.random.default_rng(17 + big)
    bases = []
    for n in ([1, 7, 40, 130] if not big else [300]):
        x = _bounded(rng, (n, n)) + 1.j * _bounded(rng, (n, n))
        bases.append(('herm%d' % n, np.triu(x, 1) + np.triu(x, 1).conj().T + np.diag(x.real.diagonal())))
    r = (rng.integers(-3, 4, (24, 3)) + 1.j * rng.integers(-3, 4, (24, 3))).astype(np.complex128)
    bases.append(('psd-rankdef', r @ r.conj().T))
    bases.append(('zero', np.zeros((5, 5), dtype=np.complex128)))
    exps = EXPS if not big else [-990, -540, -270, 0, 260, 540, 990]
    batch = _scaled_batch(bases, exps)
    mats = [A for _, _, A in batch]
    res = [(Vr, Vi, W, info) for W, Vr, Vi, info in _run_eigh_z(gpu_lib, np.random.default_rng(9), mats)]
    for (i, e, A), (Vr, Vi, W, info) in zip(batch, res):
        assert info > 0
        if e == 0:
            _check(A, W, Vr + 1.j * Vi, (bases[i][0], A.shape[0]))
    _check_equivariant(batch, res, nvec=(0, 1), nval=(2,), what='block_eigh_z')


# ---- npc ------------------------------------------------------------------------------------------------------------------

@pytest.fixture
def fake_device_eigh_z():
    """the numpy test double with the complex decompositions and the complex eigh (tests/fake_device_eigh_z.py)"""
    import fake_device_eigh_z
    lib, restore = fake_device_eigh_z.install()
    yield lib
    restore()


CHARGES = ['U1', 'Z2', 'U1xZ2']


def _leg(npc, charges, seed=0):
    """a leg of 4-6 sectors with 1-7 states each"""
    rng = np.random.default_rng(seed)
    if charges == 'U1':
        ci, qs = npc.ChargeInfo([1], ['N']), [[q] for q in range(-2, 3)]
    elif charges == 'Z2':
        ci, qs = npc.ChargeInfo([2], ['P']), [[0], [1]]
    else:
        ci, qs = npc.ChargeInfo([1, 2], ['N', 'P']), [[q, p] for q in range(-1, 2) for p in range(2)]
    sizes = rng.integers(1, 8, len(qs))
    slices = np.concatenate(([0], np.cumsum(sizes)))
    return npc.LegCharge.from_qind(ci, slices, qs, +1)


def _hermitian_on(rng, leg, drop=(), real=False):
    """dense Hermitian matrix conserving the charges of `leg` (block diagonal), sectors in `drop` set to zero"""
    q = leg.to_qflat()
    n = len(q)
    x = rng.standard_normal((n, n)) + (0. if real else 1.j * rng.standard_normal((n, n)))
    h = x + x.conj().T
    mask = np.all(q[:, None, :] == q[None, :, :], axis=2)
    for qi in drop:
        sl = leg.get_slice(qi)
        mask[sl, :] = False
        mask[:, sl] = False
    return h * mask


def _check_npc_eigh(npc, A, a, sort=None):
    W, V = npc.eigh(a, sort=sort)
    assert isinstance(V, npc.ComplexArray) and W.dtype == np.float64
    V.test_sanity()
    assert V.get_leg_labels()[-1] == 'eig'
    n = A.shape[0]
    Vd = V.to_ndarray().reshape(n, n)
    scale = max(np.linalg.norm(A), 1.)
    assert np.max(np.abs(Vd.conj().T @ Vd - np.eye(n))) <= 1e-13
    assert np.max(np.abs(A @ Vd - Vd * W)) <= 1e-13 * scale
    assert np.max(np.abs(np.sort(W) - np.linalg.eigvalsh(A))) <= 1e-13 * scale
    # charge conservation: V maps each sector of the first leg into the same sector of the eig leg
    assert np.all(V.re.qtotal == 0) and np.all(V.im.qtotal == 0)
    assert np.max(np.abs(np.sort(npc.eigvalsh(a, sort=sort)) - np.sort(W))) == 0.
    return W, V


def _npc_eigh_case(charges):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(CHARGES.index(charges))
    leg = _leg(npc, charges, CHARGES.index(charges))
    for drop in ((), (1,), tuple(range(leg.block_number - 1))):          # missing diagonal blocks
        A = _hermitian_on(rng, leg, drop)
        a = npc.ComplexArray.from_ndarray(A, [leg, leg.conj()], labels=['p', 'p*'])
        W, V = _check_npc_eigh(npc, A, a)
        for qi in drop:       # a missing block: eigenvalue 0, unit vectors
            sl = leg.get_slice(qi)
            assert np.all(W[sl] == 0.)
            assert np.array_equal(V.to_ndarray()[sl, sl], np.eye(sl.stop - sl.start))
        for sort in ('<', '>', 'm<', 'm>'):
            Ws, _ = _check_npc_eigh(npc, A, a, sort)
            for qi in range(leg.block_number):
                w = Ws[leg.get_slice(qi)]
                key = {'<': w, '>': -w, 'm<': np.abs(w), 'm>': -np.abs(w)}[sort]
                assert np.all(np.diff(key) >= 0.), sort
    # an empty imaginary part: a real Array promoted to complex
    A = _hermitian_on(rng, leg, real=True)
    a = npc.Array.from_ndarray(A.real, [leg, leg.conj()], labels=['p', 'p*']).astype(np.complex128)
    assert isinstance(a, npc.ComplexArray) and a.im.stored_blocks == 0
    _check_npc_eigh(npc, A, a)
    # legs with pipes: V is split back
    l2 = _leg(npc, charges, 10 + CHARGES.index(charges))
    pipe = npc.LegPipe([leg, l2])
    q = np.concatenate([(leg.to_qflat()[:, None, :] + l2.to_qflat()[None, :, :]).reshape(-1, leg.chinfo.qnumber)])
    q = leg.chinfo.make_valid(q)
    n = len(q)
    x = _crandn(rng, n, n)
    A = (x + x.conj().T) * np.all(q[:, None, :] == q[None, :, :], axis=2)
    a4 = npc.ComplexArray.from_ndarray(A.reshape(leg.ind_len, l2.ind_len, leg.ind_len, l2.ind_len),
                                       [leg, l2, leg.conj(), l2.conj()], labels=['a', 'b', 'a*', 'b*'])
    a = a4.combine_legs([['a', 'b'], ['a*', 'b*']], qconj=[+1, -1])
    assert pipe.ind_len == n
    W, V = _check_npc_eigh(npc, a.to_ndarray(), a)           # dense in the order of the pipe
    assert V.get_leg_labels() == ['(a.b)', 'eig']
    Vs = V.split_legs(0)                                          # the pipe splits as for a real V
    assert Vs.get_leg_labels() == ['a', 'b', 'eig']
    Vd = Vs.to_ndarray().reshape(n, n)
    assert np.max(np.abs(Vd.conj().T @ Vd - np.eye(n))) <= 1e-13
    assert np.max(np.abs(A @ Vd - Vd * W)) <= 1e-13 * np.linalg.norm(A)
    # not Hermitian: refused
    x = _crandn(rng, leg.ind_len, leg.ind_len) * np.all(leg.to_qflat()[:, None] == leg.to_qflat()[None, :], axis=2)
    with pytest.raises(NotImplementedError, match='complex Hermitian'):
        npc.eigh(npc.ComplexArray.from_ndarray(x, [leg, leg.conj()], labels=['p', 'p*']))
    H = _hermitian_on(rng, leg)
    with pytest.raises(NotImplementedError, match='complex Hermitian'):
        npc.eigvalsh(npc.ComplexArray.from_ndarray(1.j * H, [leg, leg.conj()]))


@pytest.mark.parametrize('charges', CHARGES)
def test_npc_complex_eigh(fake_device_eigh_z, charges):
    _npc_eigh_case(charges)
    assert fake_device_eigh_z.calls['block_eigh_z'] > 0


@pytest.mark.gpu
@pytest.mark.parametrize('charges', CHARGES)
def test_npc_complex_eigh_gpu(gpu_lib, charges):
    _npc_eigh_case(charges)


def test_complex_block_assignment(fake_device_eigh_z):
    """the reference's full_diag_effH writes the ground state into a zero Array: ``theta.dtype = complex128`` makes a real
    Array a ComplexArray in place, and ``get_block(.., insert=True)[:] = v`` writes through to both parts"""
    from tenpy_b200.linalg import np_conserved as npc
    leg = _leg(npc, 'U1')
    rng = np.random.default_rng(11)
    a = npc.Array.from_ndarray(_hermitian_on(rng, leg, real=True).real, [leg, leg.conj()], labels=['p', 'p*'])
    theta = a.zeros_like()
    theta.dtype = np.promote_types(np.complex128, np.float64)
    assert isinstance(theta, npc.ComplexArray) and theta.dtype == np.complex128
    assert theta.get_leg_labels() == ['p', 'p*']
    qi = np.array([2, 2])
    sl = leg.get_slice(2)
    v = _crandn(rng, sl.stop - sl.start, sl.stop - sl.start)
    blk = theta.get_block(qi, insert=True)
    blk[:] = v
    dense = theta.to_ndarray()
    assert np.array_equal(dense[sl, sl], v) and np.count_nonzero(dense) == v.size
    with pytest.raises(TypeError):
        theta.dtype = np.float64
