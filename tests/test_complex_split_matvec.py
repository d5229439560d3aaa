"""The split-order two-site matvec on complex states and Hamiltonians (`SplitOrderMatvec`): LP, W0 W1 and RP applied one
after the other to the split theta, the identity components of the environments skipped, and on dense tensors the
kernel sequence [[Lr, -Li], [Li, Lr]] . theta, b200_mid_contract2_z, Y_emb . [Rr; Ri], axpy replayed per bond.

CPU (test double of the device library): every bond of converged states against the combined order LHeff . theta .
RHeff, the kernel counts and the replay of the dense route, linearity and Hermiticity, the refusal of environments whose
identity component is not 1, and whole DMRG runs in the split order (the checks of test_complex_dmrg.py).  GPU: the
kernel against a long-double einsum at its edge shapes, the whole runs at L = 64, and a dense chain at chi = 512, where
``matvec_order='auto'`` takes the new route.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import fake_mid_contract_z
import test_complex_dmrg as tcd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, 'tests', 'dropin', 'run_dmrg_complex_split.py')
EPS = np.finfo(np.float64).eps

DM = {'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'D': 0.6, 'hz': 0.1}


@pytest.fixture
def fake_device(fake_device):
    """the test double of the device library with the numpy double of b200_mid_contract2_z"""
    return fake_mid_contract_z.install(fake_device)


def _converged(M, state, mixer, chi=24):
    """two sweeps in the combined order, then canonical form and fresh environments"""
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    psi = MPS.from_product_state(M.lat_sites, state)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': mixer, 'combine': True, 'matvec_order': 'combined',
                                          'trunc_params': {'chi_max': chi, 'svd_min': 1e-12}})
    eng.sweep()
    eng.sweep()
    eng.mixer_cleanup()
    psi.canonical_form()
    eng.env.clear()
    return eng, psi


def _cases():
    from tenpy_b200.models import SpinChain
    L = 8
    neel = ['up', 'down'] * (L // 2)
    return {
        'dm-sz': (SpinChain(dict(DM, L=L, conserve='Sz')), neel, True, False),
        'parity': (SpinChain({'L': L, 'Jx': 1.2, 'Jy': 0.8, 'Jz': 1., 'D': 0.5, 'hz': 0.3, 'conserve': 'parity'}),
                   ['up'] * L, True, False),
        'dm-dense': (SpinChain(dict(DM, L=L, conserve=None)), neel, None, False),
        # a real Hamiltonian on a complex state: theta = psi's theta (1 + 0.3i) + 0.2i (random of the same charges)
        'real-mpo-dense': (SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'hz': 0.1, 'conserve': None}), neel, None,
                           True),
        'real-mpo-sz': (SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'hz': 0.1, 'conserve': 'Sz'}), neel, True,
                        True),
    }


def _theta(H, psi, i0, make_complex, rng):
    from tenpy_b200.linalg import np_conserved as npc
    theta = H.combine_theta(psi.get_theta(i0, 2))
    if make_complex:
        noise = npc.Array.from_func(rng.standard_normal, theta.legs, qtotal=theta.qtotal,
                                    labels=theta.get_leg_labels())
        theta = theta * (1. + 0.3j) + noise * 0.2j
    return theta


def _rel(a, b):
    from tenpy_b200.linalg import np_conserved as npc
    return npc.norm(a - b) / max(npc.norm(a), 1e-300)


@pytest.mark.parametrize('case', ['dm-sz', 'parity', 'dm-dense', 'real-mpo-dense', 'real-mpo-sz'])
def test_split_equals_combined_every_bond(fake_device, case):
    """at every bond of a converged state the split order equals the combined order to 1e-11, with the identity shortcut
    on (immediate and deferred test) and off, for the Array theta and the packed Krylov vector; the shortcut is taken on
    every inner bond, and the dense route runs b200_mid_contract2_z once per call"""
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg.krylov_based import _pack
    M, state, mixer, make_complex = _cases()[case]
    eng, psi = _converged(M, state, mixer)
    assert (M.H_MPO.dtype is np.complex128) != make_complex
    dense = M.lat_sites[0].leg.chinfo.qnumber == 0
    rng = np.random.default_rng(7)
    for i0 in range(psi.L - 1):
        Hc = TwoSiteH(eng.env, i0, combine=True, matvec_order='combined')
        theta = _theta(Hc, psi, i0, make_complex, rng)
        assert theta.dtype == np.complex128
        ref = Hc.matvec(theta)
        assert ref.dtype == np.complex128
        for ident, check in ((True, 'immediate'), (True, 'deferred'), (False, 'immediate')):
            for packed in (False, True):
                Hs = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
                Hs.identity_env, Hs.identity_check = ident, check
                th = _pack(theta) if packed else theta
                n0 = fake_device.calls.get('mid_contract2_z', 0)
                got = Hs.matvec(th)
                Hs.deferred_check()
                n_z = fake_device.calls.get('mid_contract2_z', 0) - n0
                assert got.dtype == np.complex128 and got.get_leg_labels() == ref.get_leg_labels()
                assert _rel(ref, got) <= 1e-11, (case, i0, ident, check, packed, _rel(ref, got))
                inner = 0 < i0 < psi.L - 2
                if ident and inner:
                    assert Hs._id_env is True, (case, i0)
                # (the boundary bonds take the shortcut too where their MPO legs are not 1-dimensional)
                assert n_z == int(bool(ident and Hs._id_env and packed and dense)), (case, i0, ident, packed, n_z)


def test_complex_mpo_real_theta(fake_device):
    """a complex Hamiltonian on a real start vector: the Array-level route (npc.tensordot composes the complex products),
    complex128 result equal to the combined order"""
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    for case in ('dm-sz', 'dm-dense'):
        M, state, mixer, _ = _cases()[case]
        eng, psi = _converged(M, state, mixer)
        for i0 in range(psi.L - 1):
            Hc = TwoSiteH(eng.env, i0, combine=True, matvec_order='combined')
            theta = Hc.combine_theta(psi.get_theta(i0, 2))
            theta = theta.re if theta.dtype == np.complex128 else theta
            assert theta.dtype == np.float64
            Hs = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
            ref, got = Hc.matvec(theta), Hs.matvec(theta)
            assert got.dtype == np.complex128
            assert _rel(ref, got) <= 1e-11, (case, i0)


def test_dense_route_replay_linearity_hermiticity(fake_device):
    """dense complex route: one b200_mid_contract2_z per call; the second call of a bond replays the recorded sequence (no
    new contraction plan, the same result layout, the same result to 1e-14); H(z theta) = z H(theta); <x|Hy> = conj <y|Hx>"""
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.linalg.krylov_based import _pack
    M, state, mixer, _ = _cases()['dm-dense']
    eng, psi = _converged(M, state, mixer)
    rng = np.random.default_rng(3)
    for i0 in range(1, psi.L - 2):
        H = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
        theta = _pack(H.combine_theta(psi.get_theta(i0, 2)))
        n0 = fake_device.calls.get('mid_contract2_z', 0)
        a = H.matvec(theta)
        assert fake_device.calls.get('mid_contract2_z', 0) == n0 + 1 and H._dense_z is not None
        n_plan = fake_device.calls.get('tdot_plan', 0)
        c = H.matvec(theta)
        assert fake_device.calls.get('mid_contract2_z', 0) == n0 + 2 and fake_device.calls.get('tdot_plan', 0) == n_plan
        assert c.get_leg_labels() == a.get_leg_labels() and c.re._layout is a.re._layout
        assert _rel(a, c) <= 1e-14
        z = 0.7 - 1.3j
        az = H.matvec(_pack(theta * z))
        assert fake_device.calls.get('mid_contract2_z', 0) == n0 + 3
        assert _rel(a * z, az) <= 1e-13
        # Hermiticity on random complex vectors
        x, y = [_pack(npc.Array.from_func(rng.standard_normal, theta.legs, qtotal=theta.qtotal,
                                          labels=theta.get_leg_labels()) +
                      npc.Array.from_func(rng.standard_normal, theta.legs, qtotal=theta.qtotal,
                                          labels=theta.get_leg_labels()) * 1j) for _ in range(2)]
        xHy = npc.inner(x, H.matvec(y), axes='labels', do_conj=True)
        yHx = npc.inner(y, H.matvec(x), axes='labels', do_conj=True)
        scale = npc.norm(x) * npc.norm(H.matvec(y))
        assert abs(xHy - np.conj(yHx)) <= 1e-12 * scale
        assert fake_device.calls.get('mid_contract2_z', 0) == n0 + 6
    # a later visit of the bond (new effective Hamiltonian, same MPO) finds the geometry recorded: no new plan
    n_plan = fake_device.calls.get('tdot_plan', 0)
    H = TwoSiteH(eng.env, 2, combine=True, matvec_order='split')
    H.matvec(_pack(H.combine_theta(psi.get_theta(2, 2))))
    assert H._dense_z is not None and fake_device.calls.get('tdot_plan', 0) == n_plan


@pytest.mark.parametrize('case', ['dm-sz', 'dm-dense'])
def test_identity_shortcut_refused(fake_device, case):
    """LP scaled by 1 + 0.5i: Re LP[IdL] is still 1 but Im LP[IdL] is not 0.  The immediate test refuses the shortcut and
    the result equals the plain split order; the deferred test raises IdentityEnvRejected at the caller's check"""
    from tenpy_b200.algorithms.mps_common import TwoSiteH, IdentityEnvRejected
    from tenpy_b200.linalg.krylov_based import _pack
    M, state, mixer, _ = _cases()[case]
    eng, psi = _converged(M, state, mixer)
    i0 = 3
    ref_H = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
    ref_H.identity_env = False
    ref_H.LP = ref_H.LP * (1. + 0.5j)
    theta = _pack(ref_H.combine_theta(psi.get_theta(i0, 2)))
    ref = ref_H.matvec(theta)
    H = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
    H.LP = H.LP * (1. + 0.5j)
    n0 = fake_device.calls.get('mid_contract2_z', 0)
    got = H.matvec(theta)
    assert H._id_env is False and fake_device.calls.get('mid_contract2_z', 0) == n0
    assert _rel(ref, got) <= 1e-13
    H = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
    H.identity_check = 'deferred'
    H.LP = H.LP * (1. + 0.5j)
    H.matvec(theta)
    assert H._id_env is True
    with pytest.raises(IdentityEnvRejected):
        H.deferred_check()
    assert H._id_env is False
    assert _rel(ref, H.matvec(theta)) <= 1e-13


def test_deferred_rejection_restart_converges(fake_device):
    """a complex state that is not in canonical form: the engine's deferred test fails, the Lanczos iteration restarts in
    the plain split order, and the run ends at the energy of the run without the shortcut"""
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    L = 10
    M = SpinChain(dict(DM, L=L, conserve=None))
    res = {}
    for ident in (True, False):
        psi = MPS.from_product_state(M.lat_sites, ['up', 'down'] * (L // 2))
        psi._B[6] = psi._B[6] * 1.7              # RP[IdR] = 1.7^2 left of site 6
        rej0 = TwoSiteH.stats['identity_env_rejected']
        out = dmrg.run(psi, M, {'mixer': None, 'max_E_err': 1e-11, 'combine': True, 'matvec_order': 'split',
                                'diag_method': 'lanczos', 'identity_env': ident,
                                'trunc_params': {'chi_max': 20, 'svd_min': 1e-10}})
        res[ident] = (out['E'], TwoSiteH.stats['identity_env_rejected'] - rej0)
    assert res[True][1] >= 1
    assert abs(res[True][0] - res[False][0]) <= 1e-10 * abs(res[False][0])


@pytest.fixture
def split_runs(monkeypatch):
    """every `dmrg.run` of the test in the split order; the identity shortcut has to be taken"""
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import SplitOrderMatvec
    run = dmrg.run
    monkeypatch.setattr(dmrg, 'run', lambda psi, M, opts: run(psi, M, dict(opts, matvec_order='split')))
    n0 = SplitOrderMatvec.stats['identity_env_bonds']
    yield
    assert SplitOrderMatvec.stats['identity_env_bonds'] > n0


@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_gauge_split_fake(fake_device, split_runs, mixer):
    tcd._gauge_case(16, 48, mixer)


def test_dm_chain_free_fermions_split_fake(fake_device, split_runs):
    tcd._free_fermion_case(16, 64)


@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_parity_ed_split_fake(fake_device, split_runs, mixer):
    tcd._parity_case(mixer)


def _reference_available():
    from tenpy_b200 import dropin
    return dropin.reference_path() is not None


def _dropin(mode):
    out = subprocess.run([sys.executable, RUNNER, mode], capture_output=True, text=True, timeout=1800, cwd='/tmp')
    assert out.returncode == 0, out.stderr[-4000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'dmrg_complex.npz'))
    rec = got['fast_engine']
    assert rec['H_dtype'] == 'complex128' and rec['psi_dtype'] == 'complex128'
    assert abs(rec['E'] - float(gold['E'])) <= 1e-10 * abs(float(gold['E'])), (rec['E'], float(gold['E']))
    np.testing.assert_allclose(rec['S'], gold['S'], rtol=0, atol=1e-8)
    assert rec['chi'] == gold['chi'].tolist()
    assert got['identity_env_bonds'] > 0
    return got


@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_dropin_haldane_split_fake():
    """the reference's FermionicHaldaneModel through fast_two_site_engine() with the split order forced"""
    _dropin('fake')


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _dev(a):
    from tenpy_b200 import backend
    return backend.to_device(np.ascontiguousarray(a))


def _nan(n):
    import torch
    from tenpy_b200 import backend
    return torch.full((max(int(n), 1),), float('nan'), dtype=torch.float64, device=backend.device())


def _planar(z):
    return np.concatenate([z.real.ravel(), z.imag.ravel()])


@pytest.mark.gpu
@pytest.mark.parametrize('K1,K2,N1,N2,C1,outer,inner', [
    (16, 4, 16, 4, 4, 3, 255), (0, 12, 4, 8, 2, 2, 257), (12, 0, 9, 3, 3, 2, 255), (1, 0, 1, 0, 1, 2, 1),
    (8, 8, 16, 0, 8, 2, 300), (9, 8, 6, 6, 2, 3, 257), (16, 16, 48, 0, 4, 2, 100), (3, 20, 0, 9, 1, 2, 1),
    (1, 1, 1, 1, 1, 1, 1), (1, 1, 1024, 0, 1, 2, 3), (4, 4, 2, 2, 2, 66000, 1)])
def test_mid_contract2_z(gpu_lib, K1, K2, N1, N2, C1, outer, inner):
    """b200_mid_contract2_z against a long-double complex einsum: K1 + K2 in {1, 16, 17, 32} and empty segments, N up to
    1024, inner not a multiple of the 256-thread block, outer above 65535; OUT1 is the real embedding of Y, OUT2 planar;
    nothing is written outside the outputs"""
    rng = np.random.default_rng(K1 * 1000 + K2 * 100 + N1 + N2 + outer)
    K, N = K1 + K2, N1 + N2

    def cplx(*shape):
        return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    M, T1, T2 = cplx(N, K), cplx(outer, K1, inner), cplx(outer, K2, inner)
    P = N1 // C1 if N1 else 0
    s1, s2, pad = 4 * outer * N1 * inner, 2 * outer * N2 * inner, 3
    b1, b2 = _nan(s1 + 2 * pad), _nan(s2 + 2 * pad)
    gpu_lib.mid_contract2_z(K1, K2, N1, N2, C1, outer, inner, _dev(_planar(M)),
                            _dev(_planar(T1) if K1 else np.zeros(1)), _dev(_planar(T2) if K2 else np.zeros(1)),
                            b1[pad:], b2[pad:])
    from tenpy_b200 import backend
    o1, o2 = backend.to_host(b1).copy(), backend.to_host(b2).copy()
    for o, s in ((o1, s1), (o2, s2)):
        assert np.all(np.isnan(o[:pad])) and np.all(np.isnan(o[pad + s:])), 'a kernel wrote outside its output'
    T = np.concatenate([T1, T2], axis=1)
    ref = np.einsum('nk,oki->oni', M.astype(np.clongdouble), T.astype(np.clongdouble))
    den = np.einsum('nk,oki->oni', np.abs(M), np.abs(T))
    bound = 2 * (2 * K + 1) * EPS * den               # 2K chained FMAs per part, |Re|, |Im| <= |z|
    if N1:
        emb = o1[pad:pad + s1].reshape(2 * outer * P, 2 * C1 * inner)
        m, w = outer * P, C1 * inner
        Yr, Yi = emb[:m, :w], emb[m:, :w]
        assert np.array_equal(emb[m:, w:], Yr) and np.array_equal(emb[:m, w:], -Yi)
        Y = (Yr + 1j * Yi).reshape(outer, P, C1, inner).reshape(outer, N1, inner)
        assert np.all(np.abs(Y - ref[:, :N1]) <= bound[:, :N1])
    if N2:
        y = o2[pad:pad + s2]
        y = (y[:s2 // 2] + 1j * y[s2 // 2:]).reshape(outer, N2, inner)
        assert np.all(np.abs(y - ref[:, N1:]) <= bound[:, N1:])


@pytest.mark.gpu
def test_mid_contract2_z_argument_checks(gpu_lib):
    """K outside 1..32, N > 1024, C1 not dividing N1 and both planes of M above 48 KB are refused before any launch"""
    from tenpy_b200._lib import B200Error
    M, T, OUT = _nan(64), _nan(64), _nan(64)
    for K1, K2, N1, N2, C1 in ((17, 16, 1, 1, 1), (0, 0, 1, 1, 1), (-1, 2, 1, 1, 1), (1, 1, 600, 425, 1),
                               (16, 16, 48, 49, 1), (4, 4, 6, 0, 4), (4, 4, 6, 0, 0)):
        with pytest.raises(B200Error, match='error 1:'):
            gpu_lib.mid_contract2_z(K1, K2, N1, N2, C1, 1, 1, M, T, T, OUT, OUT)
    from tenpy_b200 import backend
    assert np.all(np.isnan(backend.to_host(OUT)))


@pytest.mark.gpu
@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_gauge_split_gpu(gpu_lib, split_runs, mixer):
    tcd._gauge_case(64, 128, mixer)


@pytest.mark.gpu
def test_dm_chain_free_fermions_split_gpu(gpu_lib, split_runs):
    tcd._free_fermion_case(64, 128)


@pytest.mark.gpu
@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_parity_ed_split_gpu(gpu_lib, split_runs, mixer):
    tcd._parity_case(mixer)


@pytest.mark.gpu
@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_dropin_haldane_split_gpu(gpu_lib):
    _dropin('cuda')


@pytest.mark.gpu
def test_dense_chain_auto_takes_new_route(gpu_lib, monkeypatch):
    """the DM chain without charges at chi = 512: theta's block has 2^20 elements, so 'auto' takes the dense complex
    route; one sweep with 'auto' and one with 'combined' from the same state agree in energy to 1e-10"""
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import SplitOrderMatvec
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    L, chi = 20, 512
    J, D = DM['Jx'], DM['D']
    M = SpinChain(dict(DM, L=L, conserve=None))
    Mr = SpinChain({'L': L, 'Jx': np.hypot(J, D), 'Jy': np.hypot(J, D), 'Jz': DM['Jz'], 'hz': DM['hz'], 'conserve': None})
    psi = MPS.from_product_state(Mr.lat_sites, ['up', 'down'] * (L // 2))
    trunc = {'chi_max': chi, 'svd_min': 1e-45}
    # the state is grown on the gauge-equivalent real chain and carried over by prod_j exp(-i j phi Sz_j)
    dmrg.run(psi, Mr, {'mixer': None, 'combine': True, 'trunc_params': trunc, 'chi_list': {0: 64, 2: 256, 4: chi},
                       'min_sweeps': 6, 'max_sweeps': 6, 'max_E_err': 0.})
    assert max(psi.chi) == chi
    phi = np.arctan2(D, J)
    sz = np.real(np.diag(M.lat_sites[0].get_op('Sz').to_ndarray()))
    assert SplitOrderMatvec.SPLIT_MIN_BLOCK <= chi * 2 * 2 * chi
    calls = []
    kernel = gpu_lib.mid_contract2_z
    monkeypatch.setattr(gpu_lib, 'mid_contract2_z', lambda *a: (calls.append(a[5:7]), kernel(*a))[1])
    E = {}
    for order in ('auto', 'combined'):
        Bs = [psi.get_B(j).astype(np.complex128).scale_axis(np.exp(-1j * j * phi * sz), 'p') for j in range(L)]
        state = MPS(M.lat_sites, Bs, [None if s is None else np.array(s) for s in psi._S], form=list(psi.form))
        eng = dmrg.TwoSiteDMRGEngine(state, M, {'mixer': None, 'combine': True, 'trunc_params': trunc,
                                                'matvec_order': order})
        n0 = len(calls)
        eng.sweep()
        E[order] = float(eng.update_stats['E_total'][-1])
        assert (len(calls) > n0) == (order == 'auto')
    assert (chi, chi) in calls                        # the bonds at chi_l = chi_r = chi ran the new kernel
    assert abs(E['auto'] - E['combined']) <= 1e-10 * abs(E['combined']), E
