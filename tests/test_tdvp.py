"""Real-time TDVP: the Lanczos time evolution (`LanczosEvolution`), the Krylov-combination kernel, the engine's own TDVP
driver (`tenpy_b200.algorithms.tdvp`) and the reference's TDVP engines on the drop-in.

* Drop-in (tests/dropin/run_tdvp.py, one case per child process): the UNMODIFIED reference ``TwoSiteTDVPEngine`` /
  ``SingleSiteTDVPEngine`` on the engine and ``dropin.fast_tdvp_engine()`` against the numbers of the plain reference
  (tests/golden/tdvp.npz, written by tests/golden/make_golden_tdvp.py).  Tolerances of test_tebd_real.py: observables,
  energy and norm 1e-9 absolute, entropies 1e-8, bond dimensions exactly, the Loschmidt amplitude <psi(0)|psi(t)> 1e-9 in
  modulus and phase.
* The engine's driver on the engine's models: the same goldens for the XXZ, TFI and Hubbard chains; the complex DM chain
  against the gauge-equivalent real XXZ chain; a chain at saturated bond dimension against ``expm(-i t H) psi0``.
* `LanczosEvolution` against ``scipy.linalg.expm(delta H) psi0`` on random hermitian operators, one block and charged.
* GPU: the kernel ``b200_krylov_combine_f64`` against numpy at its edge shapes, and its argument checks.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg

import fake_krylov_combine
import fake_mid_contract_z

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, 'tests', 'dropin', 'run_tdvp.py')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'tdvp.npz')
CASES = ['xxz', 'tfi', 'hub', 'nnn', 'haldane', 'xxz_1site']
DT, N_STEPS, TRUNC = 0.05, 8, {'chi_max': 64, 'svd_min': 1.e-10}


@pytest.fixture
def fake_device(fake_device):
    """the test double of the device library with the numpy doubles of b200_krylov_combine_f64 and b200_mid_contract2_z"""
    return fake_mid_contract_z.install(fake_krylov_combine.install(fake_device))


def _reference_available():
    from tenpy_b200 import dropin
    return dropin.reference_path() is not None


def _check(rec, case, gold):
    assert rec['chi'] == gold[case + '_chi'].tolist(), (case, rec['chi'])
    np.testing.assert_allclose(rec['S'], gold[case + '_S'], rtol=0, atol=1e-8, err_msg=case)
    for key in ('obs', 'E', 'norm'):
        np.testing.assert_allclose(rec[key], gold[case + '_' + key], rtol=0, atol=1e-9, err_msg=case + ' ' + key)
    amp, ref = complex(*rec['amp']), complex(*gold[case + '_amp'])
    assert abs(abs(amp) - abs(ref)) <= 1e-9, (case, amp, ref)
    assert abs(np.angle(amp / ref)) <= 1e-9, (case, amp, ref)


def _run_dropin(mode, case):
    out = subprocess.run([sys.executable, RUNNER, mode, case], capture_output=True, text=True, timeout=1800, cwd='/tmp')
    assert out.returncode == 0, out.stderr[-4000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    gold = np.load(GOLDEN)
    for arm in ('reference_engine', 'fast_engine'):
        _check(got[arm], case, gold)
    return got


@pytest.mark.parametrize('case', CASES)
@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_dropin_tdvp_host_logic(case):
    """the reference's TDVP engines and fast_tdvp_engine() on the CPU test double match the plain reference"""
    got = _run_dropin('fake', case)
    assert got['krylov_combine_calls'] > 0


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_dropin_tdvp_gpu(gpu_lib, case):
    """the same on the H100"""
    _run_dropin('cuda', case)


# ---------------------------------------------------------------------------------------------- the engine's driver
def _engine_case(name):
    from tenpy_b200.models import SpinChain, TFIChain, FermiHubbardChain
    if name == 'xxz':
        return SpinChain({'L': 10, 'Jx': 1., 'Jy': 1., 'Jz': 1.3, 'hz': 0., 'conserve': 'Sz'}), ['up', 'down'] * 5, 'Sz'
    if name == 'tfi':
        return TFIChain({'L': 10, 'J': 1., 'g': 1.2, 'conserve': None}), ['up'] * 10, 'Sz'
    return FermiHubbardChain({'L': 6, 't': 1., 'U': 3., 'mu': 0., 'cons_N': 'N', 'cons_Sz': 'Sz'}), ['up', 'down'] * 3, \
        'Ntot'


def _dense_state(psi):
    """the state vector (d, ..., d) of the engine's MPS: ``Th[0] B[1] ... B[L-1]``, times ``psi.norm``"""
    v = np.ones((1, 1), dtype=np.complex128)
    for i in range(psi.L):
        B = psi.get_B(i, 'Th' if i == 0 else 'B').transpose(['vL', 'p', 'vR']).to_ndarray()
        v = np.tensordot(v, B, axes=[[-1], [0]])
    return v[0, ..., 0] * psi.norm


def _mpo_apply(H, vec):
    """``H vec`` for the engine's finite MPO on a dense state vector"""
    L = vec.ndim
    T = np.zeros((H.get_W(0).get_leg('wL').ind_len,) + vec.shape, dtype=np.complex128)
    T[H.get_IdL(0)] = vec
    for i in range(L):
        W = H.get_W(i).transpose(['wL', 'wR', 'p', 'p*']).to_ndarray()
        T = np.tensordot(W, T, axes=[[0, 3], [0, 1 + i]])                # wR p  (T without w, p_i)
        T = np.moveaxis(T, 1, 1 + i)
    return T[H.get_IdR(L - 1)]


def _observables(M, psi, psi0, op):
    """the quantities of tests/dropin/run_tdvp.py, measured as the reference measures them: one-site expectation values
    from ``theta_i = S_i B_i`` (after single-site TDVP the stored Schmidt values are the ones to use, reference
    tdvp.py:410), energy and Loschmidt amplitude from the state vector ``Th[0] B[1] ... B[L-1]``"""
    v, v0 = _dense_state(psi), _dense_state(psi0)
    o = M.lat_sites[0].get_op(op).transpose(['p', 'p*']).to_ndarray()
    obs = []
    for i in range(psi.L):
        th = psi.get_theta(i, n=1).transpose(['vL', 'p0', 'vR']).to_ndarray()
        obs.append(float(np.real(np.vdot(th, np.einsum('pq,aqb->apb', o, th)))))
    return {'obs': obs, 'E': float(np.real(np.vdot(v, _mpo_apply(M.H_MPO, v)))), 'S': list(psi.entanglement_entropy()),
            'chi': list(psi.chi), 'norm': float(psi.norm), 'amp': [np.vdot(v0, v).real, np.vdot(v0, v).imag]}


def _engine_run(M, state, opts, single_site_steps=0):
    from tenpy_b200.algorithms.tdvp import TwoSiteTDVPEngine, SingleSiteTDVPEngine
    from tenpy_b200.networks.mps import MPS
    psi0 = MPS.from_product_state(M.lat_sites, state)
    psi = MPS.from_product_state(M.lat_sites, state)
    eng = TwoSiteTDVPEngine(psi, M, opts)
    eng.run()
    if single_site_steps:
        SingleSiteTDVPEngine(psi, M, dict(opts, N_steps=single_site_steps)).run()
    return psi0, psi, eng


@pytest.mark.parametrize('case', ['xxz', 'tfi', 'hub'])
def test_engine_driver_matches_reference(fake_device, case):
    """the engine's TwoSiteTDVPEngine (split or combined order as 'auto' picks, device-scalar Lanczos evolution, one
    krylov_combine per evolution) gives the numbers of the plain reference"""
    M, state, op = _engine_case(case)
    opts = {'dt': DT, 'N_steps': N_STEPS, 'trunc_params': dict(TRUNC)}
    psi0, psi, eng = _engine_run(M, state, opts)
    assert abs(eng.evolved_time - DT * N_STEPS) < 1e-15
    assert fake_device.calls.get('krylov_combine', 0) > 0
    _check(_observables(M, psi, psi0, op), case, np.load(GOLDEN))


def test_engine_driver_single_site(fake_device):
    """single-site TDVP on the engine after two-site steps (bond dimensions stay), against the reference's numbers"""
    M, state, op = _engine_case('xxz')
    opts = {'dt': DT, 'N_steps': 4, 'trunc_params': dict(TRUNC)}
    psi0, psi, _ = _engine_run(M, state, opts, single_site_steps=N_STEPS)
    _check(_observables(M, psi, psi0, op), 'xxz_1site', np.load(GOLDEN))


def test_engine_driver_complex_dm_chain(fake_device):
    """the DM chain (complex MPO) from the Neel state evolves like the gauge-equivalent real XXZ chain: the same <Sz>,
    entropies and energy to 1e-9"""
    from tenpy_b200.models import SpinChain
    J, D, Jz = 1., 0.6, 0.7
    opts = {'dt': DT, 'N_steps': 6, 'trunc_params': dict(TRUNC)}
    neel = ['up', 'down'] * 4
    Mc = SpinChain({'L': 8, 'Jx': J, 'Jy': J, 'Jz': Jz, 'D': D, 'conserve': 'Sz'})
    Mr = SpinChain({'L': 8, 'Jx': np.hypot(J, D), 'Jy': np.hypot(J, D), 'Jz': Jz, 'conserve': 'Sz'})
    assert Mc.H_MPO.dtype is np.complex128
    rc = _observables(Mc, *reversed(_engine_run(Mc, neel, opts)[:2]), 'Sz')
    rr = _observables(Mr, *reversed(_engine_run(Mr, neel, opts)[:2]), 'Sz')
    assert rc['chi'] == rr['chi']
    for key in ('obs', 'S', 'E'):
        np.testing.assert_allclose(rc[key], rr[key], rtol=0, atol=1e-9, err_msg=key)


def test_engine_driver_against_expm(fake_device):
    """at L = 8 with the bond dimensions saturated from the start (a random state, no charges), two-site TDVP is
    ``expm(-i t H) psi0`` up to the Lanczos and SVD tolerances: the state vectors agree to 1e-9"""
    from tenpy_b200.algorithms.tdvp import TwoSiteTDVPEngine
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.linalg.charges import LegCharge
    from tenpy_b200.models import TFIChain
    from tenpy_b200.networks.mps import MPS
    L = 8
    M = TFIChain({'L': L, 'J': 1., 'g': 1.2, 'conserve': None})
    rng = np.random.default_rng(5)
    v = rng.standard_normal(2**L)
    v /= np.linalg.norm(v)
    Bs, SVs, rest = [None] * L, [None] * (L + 1), v.reshape(-1, 1)
    SVs[0] = SVs[L] = np.ones(1)
    for i in range(L - 1, -1, -1):                      # right-canonical B from the right
        chi_r = rest.shape[1]
        m = rest.reshape(-1, 2 * chi_r)
        U, s, Vh = np.linalg.svd(m, full_matrices=False)
        Bs[i] = Vh.reshape(-1, 2, chi_r)
        rest = U * s
        if i:
            SVs[i] = s / np.linalg.norm(s)
    Bs[0] = Bs[0] * float(rest.reshape(-1)[0])
    leg_p = M.lat_sites[0].leg
    arrs = [npc.Array.from_ndarray(B, [LegCharge.from_trivial(B.shape[0]), leg_p, LegCharge.from_trivial(B.shape[2], qconj=-1)],
                                   labels=['vL', 'p', 'vR']) for B in Bs]
    psi = MPS(M.lat_sites, arrs, SVs, form='B')
    psi0 = _dense_state(psi)
    assert np.allclose(psi0.reshape(-1), v)
    t = DT * 6
    TwoSiteTDVPEngine(psi, M, {'dt': DT, 'N_steps': 6, 'trunc_params': {'chi_max': 64, 'svd_min': 1.e-14},
                               'lanczos_params': {'N_max': 40, 'P_tol': 1e-16}}).run()
    Hd = np.stack([_mpo_apply(M.H_MPO, e.reshape((2,) * L)).reshape(-1) for e in np.eye(2**L)], axis=1)
    ref = scipy.linalg.expm(-1j * t * Hd) @ v
    assert np.max(np.abs(_dense_state(psi).reshape(-1) - ref)) <= 1e-9


# ------------------------------------------------------------------------------------------------- LanczosEvolution
class _MatH:
    """a hermitian operator on npc vectors: ``matvec(v) = H . v`` for the 2-D Array `H` (labels 'p', 'p*')"""

    def __init__(self, H):
        self.H = H
        self.dtype = H.dtype

    def matvec(self, v):
        from tenpy_b200.linalg import np_conserved as npc
        return npc.tensordot(self.H, v, axes=['p*', 'p'])


def _random_hermitian(charged, cplx, seed):
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.linalg.charges import ChargeInfo, LegCharge
    rng = np.random.default_rng(seed)
    if charged:
        leg = LegCharge.from_qflat(ChargeInfo([1], ['N']), rng.integers(0, 3, size=48))
    else:
        leg = LegCharge.from_trivial(40)
    n = leg.ind_len
    A = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cplx else 0.)
    A = (A + A.conj().T) / np.sqrt(4. * n)
    q = leg.to_qflat()[:, 0] if charged else np.zeros(n, int)
    A = A * (q[:, None] == q[None, :])                 # charge-conserving
    Ctor = npc.ComplexArray if cplx else npc.Array
    H = Ctor.from_ndarray(A, [leg, leg.conj()], labels=['p', 'p*'])
    psi = rng.standard_normal(n) * (q == q[0]) * 3.
    return H, A, npc.Array.from_ndarray(psi, [leg], labels=['p']), psi


@pytest.mark.parametrize('charged', [False, True])
@pytest.mark.parametrize('delta,normalize,cplx,cplx_start', [
    (-0.1j, None, True, True), (-1j, None, True, True), (-0.5, False, False, True), (-0.5, False, True, True),
    (-1j, None, False, False), (-0.1j, None, False, False)])
def test_lanczos_evolution(fake_device, charged, delta, normalize, cplx, cplx_start):
    """``expm(delta H) psi0`` to 1e-10 relative (complex and real H, complex and real start vectors, normalised or with
    the norm); device_scalars True and False agree in N and result; one krylov_combine per run on the device route"""
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.linalg.krylov_based import LanczosEvolution
    H, A, psi, psi_np = _random_hermitian(charged, cplx, seed=int(abs(delta) * 10) + 7 * charged)
    if cplx_start:
        psi = psi * (0.6 + 0.8j)
        psi_np = psi_np * (0.6 + 0.8j)
    ref = scipy.linalg.expm(delta * A) @ psi_np
    if normalize is None:
        ref = ref / np.linalg.norm(ref)
    res = {}
    for dev in (True, False):
        opts = {'N_max': 40, 'P_tol': 1e-14, 'device_scalars': dev}
        n0 = fake_device.calls.get('krylov_combine', 0)
        lz = LanczosEvolution(_MatH(H), psi, opts)
        out, N = lz.run(delta, normalize=normalize)
        assert fake_device.calls.get('krylov_combine', 0) - n0 == (1 if dev else 0)
        got = out.to_ndarray() if out.get_leg_labels() == ['p'] else out.transpose(['p']).to_ndarray()
        assert np.linalg.norm(got - ref) <= 1e-10 * np.linalg.norm(ref), (dev, np.linalg.norm(got - ref))
        if dev:
            assert abs(lz.norm_check() - 1.) < 1e-12
        res[dev] = (N, got)
    assert res[True][0] == res[False][0]
    assert np.linalg.norm(res[True][1] - res[False][1]) <= 1e-12 * np.linalg.norm(ref)
    assert np.linalg.norm(npc.norm(psi) - np.linalg.norm(psi_np)) < 1e-12     # the start vector is left as it was


def test_lanczos_evolution_fallback_and_hermitian_flag(fake_device):
    """`reortho` and ``N_cache < N_max`` take the host assembly (no kernel), with the same result; the engine refuses
    ``hermitian=False``"""
    from tenpy_b200.linalg.krylov_based import LanczosEvolution
    from tenpy_b200.algorithms.tdvp import TwoSiteTDVPEngine
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    H, A, psi, psi_np = _random_hermitian(True, True, seed=3)
    ref = scipy.linalg.expm(-0.3j * A) @ psi_np
    ref /= np.linalg.norm(ref)
    for extra in ({'reortho': True}, {'N_cache': 10}):
        n0 = fake_device.calls.get('krylov_combine', 0)
        out, N = LanczosEvolution(_MatH(H), psi, dict({'N_max': 40, 'P_tol': 1e-14}, **extra)).run(-0.3j)
        assert fake_device.calls.get('krylov_combine', 0) == n0
        assert np.linalg.norm(out.to_ndarray() - ref) <= 1e-10
    M = SpinChain({'L': 4, 'conserve': 'Sz'})
    eng = TwoSiteTDVPEngine(MPS.from_product_state(M.lat_sites, ['up', 'down'] * 2), M,
                            {'dt': 0.05, 'N_steps': 1, 'lanczos_params': {'hermitian': False}})
    with pytest.raises(NotImplementedError, match='ArnoldiEvolution'):
        eng.run()
    with pytest.raises(NotImplementedError):
        TwoSiteTDVPEngine(MPS.from_product_state(M.lat_sites, ['up', 'down'] * 2), M,
                          {'Krylov_params': {'expansion_dim': 2}})


def test_zero_site_h(fake_device):
    """ZeroSiteH is hermitian: its matrix (to_matrix) and its matvec (<x|H y> = conj <y|H x> on random bond matrices)"""
    from tenpy_b200.algorithms.dmrg import TwoSiteDMRGEngine
    from tenpy_b200.algorithms.mps_common import ZeroSiteH
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    M = SpinChain({'L': 6, 'Jz': 1.3, 'conserve': 'Sz'})
    psi = MPS.from_product_state(M.lat_sites, ['up', 'down'] * 3)
    eng = TwoSiteDMRGEngine(psi, M, {'max_sweeps': 2, 'trunc_params': {'chi_max': 8}, 'mixer': True})
    eng.run()
    H0 = ZeroSiteH(eng.env, 3)
    Hm = H0.to_matrix().to_ndarray()
    assert Hm.shape == (H0.N, H0.N) and np.allclose(Hm, Hm.conj().T, atol=1e-12)
    rng = np.random.default_rng(2)
    legs = [H0.LP.get_leg('vR').conj(), H0.RP.get_leg('vL').conj()]
    x, y = [npc.Array.from_func(rng.standard_normal, legs, labels=['vL', 'vR']) for _ in range(2)]
    Hy = H0.matvec(y)
    assert Hy.get_leg_labels() == ['vL', 'vR']
    xHy = npc.inner(x, Hy, axes='labels', do_conj=True)
    yHx = npc.inner(y, H0.matvec(x), axes='labels', do_conj=True)
    assert abs(xHy - np.conj(yHx)) <= 1e-12 * npc.norm(x) * npc.norm(Hy)


# ------------------------------------------------------------------------------------------------------ the kernel
def _combine_inputs(nvec, n, in_planes, seed):
    from tenpy_b200 import backend
    rng = np.random.default_rng(seed)
    stride = 7
    pool = rng.standard_normal(in_planes * n + stride * nvec + 1)
    coef = rng.standard_normal(2 * nvec)
    dpool = backend.to_device(pool)
    vecs = [dpool[stride * k:stride * k + in_planes * n] for k in range(nvec)]   # distinct, overlapping inputs
    return pool, coef, dpool, vecs


@pytest.mark.gpu
@pytest.mark.parametrize('in_planes', [1, 2])
@pytest.mark.parametrize('n', [0, 1, 255, 257, 10**6 + 3])
@pytest.mark.parametrize('nvec', [1, 2, 20, 64])
def test_krylov_combine_kernel(gpu_lib, nvec, n, in_planes):
    """b200_krylov_combine_f64 against numpy (long double): both planes of the output, nothing written outside"""
    from tenpy_b200 import backend
    pool, coef, dpool, vecs = _combine_inputs(nvec, n, in_planes, seed=nvec * 7 + n % 1000 + in_planes)
    ptrs = np.array([v.data_ptr() for v in vecs], dtype=np.int64)
    pad = 3
    out = backend.to_device(np.full(2 * n + 2 * pad, np.nan))
    gpu_lib.krylov_combine(n, in_planes, ptrs, backend.to_device(ptrs), backend.to_device(coef), out[pad:])
    o = backend.to_host(out)
    assert np.all(np.isnan(o[:pad])) and np.all(np.isnan(o[pad + 2 * n:]))
    re, im = np.zeros(n, np.longdouble), np.zeros(n, np.longdouble)
    mag = np.zeros(n)
    for k in range(nvec):
        x = pool[7 * k:7 * k + in_planes * n].astype(np.longdouble)
        xr, xi = (x[:n], x[n:]) if in_planes == 2 else (x, np.zeros(n, np.longdouble))
        cr, ci = np.longdouble(coef[2 * k]), np.longdouble(coef[2 * k + 1])
        re += cr * xr - ci * xi
        im += cr * xi + ci * xr
        mag += (abs(coef[2 * k]) + abs(coef[2 * k + 1])) * (np.abs(xr) + np.abs(xi)).astype(np.float64)
    bound = 4 * nvec * np.finfo(np.float64).eps * mag + 1e-300
    assert np.all(np.abs(o[pad:pad + n] - re.astype(np.float64)) <= bound)
    assert np.all(np.abs(o[pad + n:pad + 2 * n] - im.astype(np.float64)) <= bound)


@pytest.mark.gpu
def test_krylov_combine_argument_checks(gpu_lib):
    """nvec outside 1..64, in_planes not 1 or 2, n < 0 and an output overlapping an input are refused with an error
    status, without a launch and without touching the output"""
    from tenpy_b200 import backend
    from tenpy_b200._lib import B200Error
    pool, coef, dpool, vecs = _combine_inputs(65, 100, 2, seed=1)
    ptrs = np.array([v.data_ptr() for v in vecs], dtype=np.int64)
    pdev, cdev = backend.to_device(ptrs), backend.to_device(np.concatenate([coef, coef]))
    out = backend.to_device(np.full(200, np.nan))
    gpu_lib.synchronize()
    n_launch = gpu_lib.kernel_launch_count()
    for n, in_planes, p in ((100, 2, ptrs[:0]), (100, 2, ptrs), (100, 0, ptrs[:2]), (100, 3, ptrs[:2]),
                            (-1, 2, ptrs[:2])):
        with pytest.raises(B200Error, match='error 1:'):
            gpu_lib.krylov_combine(n, in_planes, p, pdev, cdev, out)
    alias = np.array([ptrs[0], out.data_ptr() + 8 * 150], dtype=np.int64)
    with pytest.raises(B200Error, match='error 1:'):
        gpu_lib.krylov_combine(100, 1, alias, backend.to_device(alias), cdev, out)
    with pytest.raises(B200Error, match='error 1:'):                   # out is an input
        gpu_lib.krylov_combine(50, 2, np.array([dpool.data_ptr()], np.int64), pdev, cdev, dpool)
    assert gpu_lib.kernel_launch_count() == n_launch
    assert np.all(np.isnan(backend.to_host(out)))
    gpu_lib.krylov_combine(0, 2, ptrs[:3], pdev, cdev, out)              # n = 0: nothing to do, no launch
    assert gpu_lib.kernel_launch_count() == n_launch


@pytest.mark.gpu
@pytest.mark.parametrize('charged', [False, True])
def test_lanczos_evolution_gpu(gpu_lib, charged):
    """LanczosEvolution on the H100 against expm, both routes"""
    from tenpy_b200.linalg.krylov_based import LanczosEvolution
    H, A, psi, psi_np = _random_hermitian(charged, True, seed=11)
    ref = scipy.linalg.expm(-1j * A) @ psi_np
    ref /= np.linalg.norm(ref)
    outs = {}
    for dev in (True, False):
        out, N = LanczosEvolution(_MatH(H), psi, {'N_max': 40, 'P_tol': 1e-14, 'device_scalars': dev}).run(-1j)
        got = out.to_ndarray()
        assert np.linalg.norm(got - ref) <= 1e-10, np.linalg.norm(got - ref)
        outs[dev] = (N, got)
    assert outs[True][0] == outs[False][0]


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['xxz', 'tfi', 'hub'])
def test_engine_driver_gpu(gpu_lib, case):
    """the engine's TwoSiteTDVPEngine on the H100 against the reference's numbers"""
    M, state, op = _engine_case(case)
    psi0, psi, _ = _engine_run(M, state, {'dt': DT, 'N_steps': N_STEPS, 'trunc_params': dict(TRUNC)})
    _check(_observables(M, psi, psi0, op), case, np.load(GOLDEN))
