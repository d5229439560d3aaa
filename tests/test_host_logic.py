"""CPU tests of the HOST logic of tenpy_b200 (no GPU): charge bookkeeping, block layouts, index plans, the
contraction-plan builder of the C library (host code), the C-ABI symbol table and the DMRG driver.

Device calls go to the numpy TEST DOUBLE of tests/fake_device.py (fixture `fake_device`): these tests check
that the host side produces the reference's block structure bit-for-bit (qdata, legs, slices, q_map) against
the golden vectors; the floating point kernels themselves are tested on the GPU (tests/test_gpu_*.py)."""
import ctypes
import os
import re

import numpy as np
import pytest

import helpers as h
from oracle import npc_blocks as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_c_abi_exports_every_declared_symbol():
    """the shared library loads without a GPU and exports every function declared in include/b200npc.h"""
    from tenpy_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'b200npc.h')).read()
    header = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
    declared = set(re.findall(r'\b(b200_[a-z0-9_]+)\s*\(', header))
    assert declared, 'no declarations found'
    cdll = _lib.load_library()
    for name in sorted(declared):
        assert hasattr(cdll, name), 'libb200npc.so does not export ' + name
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    assert cdll.b200_abi_version() == 1


def test_product_fails_loudly_without_gpu():
    """no CPU fallback: constructing the real device library without a CUDA device raises"""
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from tenpy_b200._lib import DeviceLib, B200Error
    with pytest.raises(B200Error):
        DeviceLib()


def test_host_integer_helpers():
    from tenpy_b200 import _lib
    c = _lib.load_library()
    rng = np.random.default_rng(0)
    rows = rng.integers(0, 3, size=(50, 3)).astype(np.int64)
    perm = np.zeros(50, dtype=np.int64)
    assert c.b200_lexsort_rows(rows.ctypes.data_as(_lib.c_i64p), 50, 3, perm.ctypes.data_as(_lib.c_i64p)) == 0
    assert np.array_equal(perm, np.lexsort(rows.T))
    srt = np.ascontiguousarray(rows[perm])
    out = np.zeros(51, dtype=np.int64)
    n_out = ctypes.c_int64()
    assert c.b200_find_row_differences(srt.ctypes.data_as(_lib.c_i64p), 50, 3, out.ctypes.data_as(_lib.c_i64p),
                                       ctypes.byref(n_out)) == 0
    assert np.array_equal(out[:n_out.value], ob.find_row_differences(srt))
    ch = rng.integers(-7, 8, size=(20, 3)).astype(np.int64)
    mod = np.array([1, 3, 4], dtype=np.int64)
    ref = ob.make_valid(mod, ch)
    assert c.b200_make_valid(ch.ctypes.data_as(_lib.c_i64p), 20, 3, mod.ctypes.data_as(_lib.c_i64p)) == 0
    assert np.array_equal(ch, ref)
    bs = np.array([2, 0, 3, 1], dtype=np.int64)
    mb = np.zeros(6, dtype=np.int64)
    assert c.b200_map_blocks(bs.ctypes.data_as(_lib.c_i64p), 4, mb.ctypes.data_as(_lib.c_i64p)) == 0
    assert np.array_equal(mb, [0, 0, 2, 2, 2, 3])


def test_legpipe_tables_match_reference():
    """LegPipe charges / slices / q_map equal the reference's (golden: pipes of the XXZ effective H)"""
    g = h.load('dmrg.npz')
    from tenpy_b200.linalg.charges import ChargeInfo, LegCharge, LegPipe
    mod = g['xxz_LHeff_mod']
    chinfo = ChargeInfo(list(mod))
    for prefix in ('xxz_LHeff_leg0', 'xxz_RHeff_leg2', 'xxz_theta_leg0', 'xxz_theta_leg1'):
        n = int(g[prefix + '_pipe_nlegs'])
        subs = [LegCharge.from_qind(chinfo, g[prefix + '_sub%d_slices' % j], g[prefix + '_sub%d_charges' % j],
                                    int(g[prefix + '_sub%d_qconj' % j])) for j in range(n)]
        pipe = LegPipe(subs, qconj=int(g[prefix + '_qconj']))
        assert np.array_equal(pipe.slices, g[prefix + '_slices'])
        assert np.array_equal(pipe.charges, g[prefix + '_charges'])
        assert np.array_equal(pipe.q_map, g[prefix + '_pipe_qmap'])
        assert np.array_equal(pipe.q_map_slices, g[prefix + '_pipe_qmap_slices'])


def test_array_ops_structure_vs_golden(fake_device):
    """block tables produced by the host logic are identical to the reference's"""
    from tenpy_b200.linalg import np_conserved as npc
    g = h.load('tensordot.npz')
    for ci in range(int(g['ncases'])):
        oa, obb, oc = (h.oarray_from(g, 'c%d_%s' % (ci, k)) for k in 'abc')
        a, b = h.to_product(oa), h.to_product(obb)
        a.test_sanity()
        c = npc.tensordot(a, b, axes=int(g['c%d_naxes' % ci]))
        c.test_sanity()
        h.assert_close(h.to_oracle(c), oc, 1e-13)
        a2 = h.to_product(h.oarray_from(g, 'c%d_a2' % ci))
        assert abs(npc.inner(a, a2, 'range', do_conj=True) - g['c%d_inner_aa2' % ci]) < 1e-12
        h.assert_close(h.to_oracle(a + a2 * 0.37), h.oarray_from(g, 'c%d_sum' % ci), 1e-14)
    g = h.load('reshape_svd.npz')
    a = h.to_product(h.oarray_from(g, 'a'))
    comb = a.combine_legs([['vL', 'p0'], ['p1', 'vR']], qconj=[+1, -1])
    h.assert_close(h.to_oracle(comb), h.oarray_from(g, 'comb'), 0.)
    assert comb.get_leg_labels() == ['(vL.p0)', 'w', '(p1.vR)']
    comb2 = a.combine_legs([['vR', 'p1'], ['p0', 'vL']], new_axes=[0, 2], qconj=[-1, +1])
    h.assert_close(h.to_oracle(comb2), h.oarray_from(g, 'comb2'), 0.)
    h.assert_close(h.to_oracle(comb.split_legs()), h.oarray_from(g, 'split'), 0.)
    h.assert_close(h.to_oracle(a.transpose(['p1', 'vL', 'w', 'vR', 'p0'])), h.oarray_from(g, 'transp'), 0.)
    m = h.to_product(h.oarray_from(g, 'm'))
    U, S, VH = npc.svd(m, inner_labels=['vR', 'vL'])
    h.assert_same_structure(h.to_oracle(U), h.oarray_from(g, 'm_U'))
    h.assert_same_structure(h.to_oracle(VH), h.oarray_from(g, 'm_VH'))
    U2, S2, VH2 = npc.svd(m, qtotal_LR=[[1, 1], None], inner_qconj=-1)
    h.assert_same_structure(h.to_oracle(U2), h.oarray_from(g, 'm_U2'))
    from tenpy_b200.linalg.truncation import svd_theta
    Ut, St, VHt, err, renorm = svd_theta(m, {'chi_max': 17, 'svd_min': 1e-8}, inner_labels=['vR', 'vL'])
    h.assert_same_structure(h.to_oracle(Ut), h.oarray_from(g, 'm_Ut'))
    assert np.max(np.abs(St - g['m_St'])) < 1e-13 and abs(renorm - g['m_renorm']) < 1e-13
    mp = m.copy()
    mp.iproject(g['proj_mask'], 1)
    h.assert_close(h.to_oracle(mp), h.oarray_from(g, 'm_proj'), 0.)
    h.assert_close(h.to_oracle(m.scale_axis(g['scale_s'], 0)), h.oarray_from(g, 'm_scaled'), 1e-15)
    rho = h.to_product(h.oarray_from(g, 'rho'))
    w, V = npc.eigh(rho)
    h.assert_same_structure(h.to_oracle(V), h.oarray_from(g, 'rho_V'))
    assert np.max(np.abs(w - g['rho_w'])) < 1e-12


def test_two_site_matvec_structure(fake_device):
    from tenpy_b200.linalg import np_conserved as npc
    g = h.load('dmrg.npz')
    LHeff, RHeff, theta = (h.to_product(h.oarray_from(g, 'xxz_' + k)) for k in ('LHeff', 'RHeff', 'theta'))
    assert LHeff.get_leg_labels() == ['(vR*.p0)', 'wR', '(vR.p0*)']
    t = npc.tensordot(LHeff, theta, axes=['(vR.p0*)', '(vL.p0)'])
    t = npc.tensordot(t, RHeff, axes=[['wR', '(p1.vR)'], ['wL', '(p1*.vL)']])
    h.assert_close(h.to_oracle(t), h.oarray_from(g, 'xxz_Htheta'), 1e-13)
    # plan introspection: the GEMM list equals the oracle's list (what the reference hands to CblasGemmBatch)
    from tenpy_b200.linalg.np_conserved import _PLAN_CACHE
    n_pairs = sum(p[2].n_pairs for p in _PLAN_CACHE.values())
    o1 = ob.gemm_list(h.oarray_from(g, 'xxz_LHeff'), h.oarray_from(g, 'xxz_theta'), 1)
    assert n_pairs >= len(o1)


def test_truncate_matches_reference():
    from tenpy_b200.linalg.truncation import truncate
    g = h.load('reshape_svd.npz')
    opts = [dict(chi_max=10), dict(chi_max=30, svd_min=1e-4), dict(chi_max=100, trunc_cut=1e-3),
            dict(chi_max=12, chi_min=5, degeneracy_tol=1e-2)]
    for k, o in enumerate(opts):
        mask, nn, err = truncate(g['trunc_S'], o)
        assert np.array_equal(mask, g['trunc%d_mask' % k])
        assert abs(err.eps - g['trunc%d_err' % k]) < 1e-15


def _run_dmrg(model, p_state, opts):
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    psi = MPS.from_product_state(model.lat_sites, p_state)
    res = dmrg.run(psi, model, opts)
    return res, psi


def test_dmrg_driver_tfi(fake_device):
    """driver logic (schedule, environments, Lanczos, truncation) on BASELINE config 1; golden E from reference"""
    from tenpy_b200.models import TFIChain
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    res, psi = _run_dmrg(M, ['up'] * 20, {'mixer': None, 'max_E_err': 1e-10, 'combine': True,
                                         'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['tfi_S'])) < 1e-8
    assert np.max(psi.isometry_test()) < 1e-12


def test_dmrg_driver_charges_and_mixer(fake_device):
    from tenpy_b200.models import SpinChain, FermiHubbardChain
    g = h.load('dmrg.npz')
    L = 16
    M = SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
    opts = {'mixer': True, 'mixer_params': {'amplitude': 1e-5, 'decay': 2., 'disable_after': 6}, 'max_E_err': 1e-11,
            'max_S_err': 1e-8, 'trunc_params': {'chi_max': 60, 'svd_min': 1e-10}, 'combine': True, 'max_sweeps': 20}
    res, psi = _run_dmrg(M, ['up', 'down'] * (L // 2), opts)
    assert abs(res['E'] - g['xxz_E']) < 1e-10 * abs(g['xxz_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['xxz_S'])) < 1e-7
    L = 6
    M = FermiHubbardChain({'L': L, 't': 1., 'U': 4., 'mu': 0.})
    opts['trunc_params'] = {'chi_max': 64, 'svd_min': 1e-10}
    res, psi = _run_dmrg(M, ['up', 'down'] * (L // 2), opts)
    assert abs(res['E'] - g['hub_E']) < 1e-10 * abs(g['hub_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['hub_S'])) < 1e-7


def test_mpo_matches_reference(fake_device):
    """the hand-written Hubbard MPO tensor equals the reference's W (same leg charges, same entries)"""
    from tenpy_b200.models import FermiHubbardChain
    g = h.load('dmrg.npz')
    M = FermiHubbardChain({'L': 6, 't': 1., 'U': 4., 'mu': 0.})
    W = M.H_MPO.get_W(2)
    ref = h.oarray_from(g, 'hub_W')
    got = h.to_oracle(W)
    # the reference orders its MPO states differently (graph construction); compare invariants:
    assert got.shape == ref.shape
    assert abs(np.linalg.norm(got.to_dense()) - np.linalg.norm(ref.to_dense())) < 1e-12


def test_svd_extensions_host_logic(fake_device):
    """warm start (`guess`), deflation tolerance and `n_keep`: results stay a valid SVD / valid isometries"""
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(11)
    g = h.load('reshape_svd.npz')
    m = h.to_product(h.oarray_from(g, 'm'))
    U0, S0, VH0 = npc.svd(m, inner_labels=['vR', 'vL'])
    # a nearby matrix, decomposed with the previous vectors as guess
    pert = h.to_product(h.oarray_from(g, 'm'))
    pert.iscale_prefactor(1e-3)
    m2 = m + pert
    used = npc.svd_stats.get('guess_used', 0)
    U, S, VH = npc.svd(m2, inner_labels=['vR', 'vL'], guess=(U0, VH0))
    rec = npc.tensordot(U.scale_axis(S, 1), VH, axes=1)
    assert npc.norm(rec - m2) < 1e-12 * npc.norm(m2)
    Sd = np.linalg.svd(m2.to_ndarray(), compute_uv=False)
    assert np.max(np.abs(np.sort(S)[::-1] - Sd[:len(S)])) < 1e-12
    # rank deficient matrix: deflation + completion, all vectors vs only n_keep of them
    A = rng.standard_normal((40, 12)) @ rng.standard_normal((12, 50))
    a = npc.Array.from_ndarray_trivial(A, labels=['a', 'b'])
    U, S, VH = npc.svd(a)
    k = 40
    assert np.max(np.abs(U.to_ndarray().T @ U.to_ndarray() - np.eye(k))) < 1e-12
    assert np.max(np.abs(VH.to_ndarray() @ VH.to_ndarray().T - np.eye(k))) < 1e-12
    assert np.max(np.abs(U.to_ndarray() @ np.diag(S) @ VH.to_ndarray() - A)) < 1e-12 * np.linalg.norm(A)
    U, S, VH = npc.svd(a, n_keep=20)
    Vd = VH.to_ndarray()
    assert np.max(np.abs(Vd[:20] @ Vd[:20].T - np.eye(20))) < 1e-12 and np.all(Vd[20:] == 0.) and np.all(S[20:] == 0.)
    assert np.all(S[12:20] > 0.)
    # deflation tolerance: directions below 1e-6 |A| are replaced, the factorisation error stays below it
    q1, _ = np.linalg.qr(rng.standard_normal((30, 30)))
    q2, _ = np.linalg.qr(rng.standard_normal((30, 30)))
    s = np.logspace(0, -12, 30)
    B = (q1 * s) @ q2
    b = npc.Array.from_ndarray_trivial(B)
    U, S, VH = npc.svd(b, deflation_tol=1e-6)
    assert np.max(np.abs(S - s)) < 2e-6
    assert np.max(np.abs(U.to_ndarray() @ np.diag(S) @ VH.to_ndarray() - B)) < 1e-5
    assert np.max(np.abs(VH.to_ndarray() @ VH.to_ndarray().T - np.eye(30))) < 1e-12


def test_matvec_split_order_equals_combined(fake_device):
    """`TwoSiteH.matvec` in the 'split' contraction order (LP, W0 W1, RP on the split theta; d times fewer flops)
    returns the same Array as the reference's combined sequence LHeff . theta . RHeff -- dense, U(1) and U(1)xU(1), and
    dense with K = D d^2 = 96 > 32, where W0 W1 is applied by npc.tensordot instead of the streaming kernel"""
    from tenpy_b200.models import TFIChain, SpinChain, FermiHubbardChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    dense_hubbard = FermiHubbardChain({'L': 6, 't': 1., 'U': 4., 'mu': 0., 'cons_N': None, 'cons_Sz': None})
    cases = [(TFIChain({'L': 8, 'J': 1., 'g': 1.1, 'conserve': None}), ['up'] * 8, None),
             (SpinChain({'L': 8, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'conserve': 'Sz'}), ['up', 'down'] * 4, True),
             (FermiHubbardChain({'L': 6, 't': 1., 'U': 4., 'mu': 0.}), ['up', 'down'] * 3, True),
             (dense_hubbard, ['up', 'down'] * 3, None)]
    for M, state, mixer in cases:
        psi = MPS.from_product_state(M.lat_sites, state)
        eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': mixer, 'combine': True, 'matvec_order': 'combined',
                                              'trunc_params': {'chi_max': 24, 'svd_min': 1e-12}})
        eng.sweep()
        eng.sweep()
        L = psi.L
        for i0 in range(L - 1):
            Hc = TwoSiteH(eng.env, i0, combine=True, matvec_order='combined')
            Hs = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
            Hs.identity_env = False      # the contraction order alone (the identity shortcut: test_matvec_identity_env_routes)
            theta = Hc.combine_theta(psi.get_theta(i0, 2))
            n_mid = fake_device.calls.get('mid_contract', 0)
            a, b = Hc.matvec(theta), Hs.matvec(theta)
            if M is dense_hubbard:
                assert fake_device.calls.get('mid_contract', 0) == n_mid
            assert a.get_leg_labels() == b.get_leg_labels()
            assert npc.norm(a - b) <= 1e-13 * max(npc.norm(a), 1e-300)
        # 'auto' picks the combined order for these small blocks, and 'split' once the threshold is lowered
        Ha = TwoSiteH(eng.env, L // 2 - 1, combine=True)
        th = Ha.combine_theta(psi.get_theta(L // 2 - 1, 2))
        assert not Ha._use_split(th)
        Ha.SPLIT_MIN_BLOCK = 1
        assert Ha._use_split(th)


def test_dmrg_driver_split_matvec(fake_device):
    """the whole DMRG run with matvec_order='split' reproduces the reference goldens (TFI config 1 and XXZ-Sz)"""
    from tenpy_b200.models import TFIChain, SpinChain
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    res, psi = _run_dmrg(M, ['up'] * 20, {'mixer': None, 'max_E_err': 1e-10, 'combine': True, 'matvec_order': 'split',
                                         'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['tfi_S'])) < 1e-8
    L = 16
    M = SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
    opts = {'mixer': True, 'mixer_params': {'amplitude': 1e-5, 'decay': 2., 'disable_after': 6}, 'max_E_err': 1e-11,
            'max_S_err': 1e-8, 'trunc_params': {'chi_max': 60, 'svd_min': 1e-10}, 'combine': True, 'max_sweeps': 20,
            'matvec_order': 'split'}
    res, psi = _run_dmrg(M, ['up', 'down'] * (L // 2), opts)
    assert abs(res['E'] - g['xxz_E']) < 1e-10 * abs(g['xxz_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['xxz_S'])) < 1e-7


def test_matvec_fused_mid_contract(fake_device):
    """split-order matvec on dense (one block) tensors with K = D d^2 <= 32: W0.W1 is applied to the middle legs by
    b200_mid_contract_f64 in one streaming pass; equals LP . theta . (W0 W1) . RP contracted by npc.tensordot"""
    from tenpy_b200.models import TFIChain, SpinChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    M = TFIChain({'L': 8, 'J': 1., 'g': 1.1, 'conserve': None})
    psi = MPS.from_product_state(M.lat_sites, ['up'] * 8)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': None, 'combine': True, 'trunc_params': {'chi_max': 24, 'svd_min': 1e-12}})
    eng.sweep()
    eng.sweep()
    for i0 in range(7):
        Hf = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
        Hf.identity_env = False      # b200_mid_contract_f64 (the two-segment kernel: identity test)
        theta = Hf.combine_theta(psi.get_theta(i0, 2))
        a = npc.tensordot(Hf.LP, theta.split_legs(['(vL.p0)', '(p1.vR)']), axes=['vR', 'vL'])
        a = npc.tensordot(a, npc.tensordot(Hf.W0, Hf.W1, axes=['wR', 'wL']),
                          axes=[['wR', 'p0', 'p1'], ['wL', 'p0*', 'p1*']])
        a = npc.tensordot(a, Hf.RP, axes=[['vR', 'wR'], ['vL', 'wL']]).ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
        a = a.combine_legs([['vL', 'p0'], ['p1', 'vR']], pipes=[Hf.pipeL, Hf.pipeR]).itranspose(theta.get_leg_labels())
        n0 = fake_device.calls.get('mid_contract', 0)
        b = Hf.matvec(theta)
        assert fake_device.calls.get('mid_contract', 0) == n0 + 1
        assert a.get_leg_labels() == b.get_leg_labels()
        assert npc.norm(a - b) <= 1e-13 * max(npc.norm(a), 1e-300)
    # whole runs: dense, and with charges, where the streaming kernel is never taken
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    res, psi = _run_dmrg(M, ['up'] * 20, {'mixer': None, 'max_E_err': 1e-10, 'combine': True, 'matvec_order': 'split',
                                         'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    M = SpinChain({'L': 8, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
    n0 = fake_device.calls.get('mid_contract', 0)
    _run_dmrg(M, ['up', 'down'] * 4, {'mixer': True, 'matvec_order': 'split', 'max_sweeps': 3,
                                     'trunc_params': {'chi_max': 16, 'svd_min': 1e-10}})
    assert fake_device.calls.get('mid_contract', 0) == n0


def test_lanczos_device_scalars(fake_device):
    """Lanczos with device-resident (alpha, beta) read back in chunks stops at the same Krylov dimension and returns the
    same vector as the host-scalar loop: fixed N (the benchmark setting), early convergence inside a chunk, breakdown
    (start vector = eigenvector), and whole DMRG runs"""
    from tenpy_b200.models import TFIChain, SpinChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg.krylov_based import LanczosGroundState
    from tenpy_b200.linalg import np_conserved as npc
    M = SpinChain({'L': 10, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'conserve': 'Sz'})
    psi = MPS.from_product_state(M.lat_sites, ['up', 'down'] * 5)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': True, 'trunc_params': {'chi_max': 20, 'svd_min': 1e-12}})
    eng.sweep()
    eng.sweep()
    H = TwoSiteH(eng.env, 4, combine=True)
    rng = np.random.default_rng(2)
    theta0 = H.combine_theta(psi.get_theta(4, 2))
    noise = npc.Array.from_func(rng.standard_normal, theta0.legs, qtotal=theta0.qtotal, labels=theta0.get_leg_labels())
    start = theta0 + noise * 0.3
    for opts in ({'N_min': 10, 'N_max': 10}, {'N_min': 2, 'N_max': 20, 'P_tol': 1e-8}, {'N_min': 3, 'N_max': 20},
                 {'N_min': 2, 'N_max': 20, 'sync_every': 5, 'P_tol': 1e-6}):
        E0, v0, N0 = LanczosGroundState(H, start.copy(deep=True), dict(opts)).run()
        n_before = fake_device.calls.get('lanczos_update_dev', 0)
        E1, v1, N1 = LanczosGroundState(H, start.copy(deep=True), dict(opts, device_scalars=True)).run()
        assert fake_device.calls.get('lanczos_update_dev', 0) >= n_before + N0
        assert N1 == N0 and abs(E1 - E0) < 1e-13 * max(1., abs(E0))
        assert npc.norm(v1 - v0) < 1e-12
    # breakdown: the exact ground state of the block as start vector
    Eg, vg, _ = LanczosGroundState(H, start.copy(deep=True), {'N_min': 2, 'N_max': 40, 'P_tol': 1e-28}).run()
    for dev in (False, True):
        E2, v2, N2 = LanczosGroundState(H, vg.copy(deep=True), {'N_min': 2, 'N_max': 12, 'device_scalars': dev}).run()
        assert abs(E2 - Eg) < 1e-12 and abs(abs(npc.inner(v2, vg, axes='range', do_conj=True)) - 1.) < 1e-12
        assert np.all(np.isfinite(v2.to_ndarray()))
    # whole runs
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    res, psi = _run_dmrg(M, ['up'] * 20, {'mixer': None, 'max_E_err': 1e-10, 'combine': True,
                                         'lanczos_params': {'device_scalars': True},
                                         'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['tfi_S'])) < 1e-8


def test_block_svd_retries_once_after_noconv():
    """binding logic: B200_ERR_NOCONV of the block SVD is answered by ONE repetition with the conservative settings (four
    inner sweeps of the pivot solver, no deflation, zeroed outputs), the library state is restored, a second failure raises"""
    import torch
    from tenpy_b200 import _lib

    class FakeC:
        def __init__(self, rcs):
            self.rcs, self.calls, self.state, self.log = list(rcs), 0, {'inner': 2, 'defl': 1}, []

        def b200_block_svd_worksize(self, nb, m, n):
            return 64

        def b200_block_svd_f64(self, *a):
            self.calls += 1
            self.log.append(dict(self.state))
            return self.rcs.pop(0)

        def b200_svd_set_eig_inner_sweeps(self, n):
            old, self.state['inner'] = self.state['inner'], n
            return old

        def b200_svd_set_deflation(self, on):
            old, self.state['defl'] = self.state['defl'], on
            return old

        def b200_last_error(self):
            return b'block Jacobi SVD did not converge'

    def make(rcs):
        lib = object.__new__(_lib.DeviceLib)
        lib.torch, lib.c, lib.device, lib.profile, lib._stream, lib.noconv_retries = torch, FakeC(rcs), torch.device('cpu'), None, \
            _lib.c_vp(0), 0
        return lib
    A, U, S, VT = torch.ones(4, dtype=torch.float64), torch.ones(4, dtype=torch.float64), torch.zeros(2, dtype=torch.float64), \
        torch.ones(4, dtype=torch.float64)
    lib = make([_lib.B200_ERR_NOCONV, 0])
    lib.block_svd([2], [2], [0], [0], [0], [0], A, U, S, VT)
    assert lib.c.calls == 2 and lib.noconv_retries == 1
    assert lib.c.log == [{'inner': 2, 'defl': 1}, {'inner': 4, 'defl': 0}] and lib.c.state == {'inner': 2, 'defl': 1}
    assert float(U.abs().sum()) == 0. and float(VT.abs().sum()) == 0. and float(A.sum()) == 4.
    lib = make([_lib.B200_ERR_NOCONV, _lib.B200_ERR_NOCONV])
    with pytest.raises(_lib.B200Error):
        lib.block_svd([2], [2], [0], [0], [0], [0], A, U, S, VT)
    assert lib.c.calls == 2 and lib.c.state == {'inner': 2, 'defl': 1}
    lib = make([0])
    lib.block_svd([2], [2], [0], [0], [0], [0], A, U, S, VT)
    assert lib.c.calls == 1 and lib.noconv_retries == 0


def test_svd_theta_completes_only_what_the_truncation_can_keep(fake_device):
    """numerically rank-deficient theta: the directions the SVD kernel deflates get an orthonormal completion only if the
    truncation could keep them -- not with svd_min above the deflation threshold (they are cut: zero vectors, S = 0), but with
    a tiny svd_min (the benchmark harness: 1e-45), where the reference keeps LAPACK's ~1e-17 values and chi stays at chi_max"""
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.linalg.truncation import svd_theta
    rng = np.random.default_rng(3)
    n, r = 24, 5
    q1, _ = np.linalg.qr(rng.standard_normal((n, r)))
    q2, _ = np.linalg.qr(rng.standard_normal((n, r)))
    A = (q1 * np.logspace(0, -3, r)) @ q2.T
    ci = npc.ChargeInfo()
    legs = [npc.LegCharge.from_trivial(n, ci, +1), npc.LegCharge.from_trivial(n, ci, -1)]

    def run(trunc):
        theta = npc.Array.from_ndarray(A, legs, labels=['(vL.p0)', '(p1.vR)'])
        before = fake_device.calls.get('col_sqnorms', 0)          # the leverage scores: first step of every completion
        U, S, VH, err, renorm = svd_theta(theta, trunc)
        return U, S, VH, fake_device.calls.get('col_sqnorms', 0) - before
    U, S, VH, completed = run({'chi_max': 16, 'svd_min': 1e-10})
    assert completed == 0 and len(S) == r
    assert np.max(np.abs(npc.tensordot(U.scale_axis(S, 1), VH, axes=1).to_ndarray() * np.linalg.norm(A) - A)) < 1e-12
    U, S, VH, completed = run({'chi_max': 16, 'svd_min': 1e-45, 'trunc_cut': None, 'svd_deflation_tol': 1e-10})
    assert completed == 1 and len(S) == 16
    u, vh = U.to_ndarray(), VH.to_ndarray()
    assert np.max(np.abs(u.T @ u - np.eye(16))) < 1e-12 and np.max(np.abs(vh @ vh.T - np.eye(16))) < 1e-12
    U, S, VH, completed = run({'chi_max': 16, 'svd_min': 1e-14})      # below the rounding-level threshold: completed as well
    assert completed == 1


def test_sweep_resolves_device_statistics(fake_device):
    """the overlap statistic and the norm of the Lanczos result stay on the device during a sweep (no host round trip between
    the eigensolver and the SVD); `sweep` reads them in one transfer: `update_stats['ov_change']` holds numbers afterwards"""
    from tenpy_b200.models import TFIChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    M = TFIChain({'L': 8, 'J': 1., 'g': 1.2, 'conserve': None})
    psi = MPS.from_product_state(M.lat_sites, ['up'] * 8)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': None, 'combine': True, 'diag_method': 'lanczos',
                                           'trunc_params': {'chi_max': 16, 'svd_min': 1e-12}})
    eng.sweep()
    eng.sweep()
    ov = np.array(eng.update_stats['ov_change'], dtype=float)
    assert len(ov) == 2 * 2 * (8 - 2) and np.all(np.isfinite(ov)) and np.all(ov > -1e-12) and np.all(ov <= 1. + 1e-12)
    assert ov[-1] < 1e-6                      # converged: the last update hardly changes the wave function
    assert eng._pending_scalars == []


def test_split_matvec_shares_buffers_without_charges(fake_device):
    """the split-order matvec relabels instead of copying when combining / splitting is the identity on the packed buffer
    (no charges): no block-move launch for the theta reshapes, input untouched, result owns its buffer"""
    from tenpy_b200.models import TFIChain, SpinChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    M = TFIChain({'L': 8, 'J': 1., 'g': 1.1, 'conserve': None})
    psi = MPS.from_product_state(M.lat_sites, ['up'] * 8)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': None, 'combine': True, 'trunc_params': {'chi_max': 24, 'svd_min': 1e-12}})
    eng.sweep()
    eng.sweep()
    H = TwoSiteH(eng.env, 3, combine=True, matvec_order='split')
    H.identity_env = False
    theta = H.combine_theta(psi.get_theta(3, 2))
    before = theta.to_ndarray().copy()
    H.matvec(theta)                                   # plans cached now
    n0 = fake_device.calls.get('copy_blocks', 0)
    out = H.matvec(theta)
    n_copies = fake_device.calls.get('copy_blocks', 0) - n0
    ref = TwoSiteH(eng.env, 3, combine=True, matvec_order='combined').matvec(theta)
    assert npc.norm(out - ref) < 1e-13 * npc.norm(ref)
    assert np.array_equal(theta.to_ndarray(), before)
    assert out._buf.data_ptr() != theta._buf.data_ptr()
    # LHeff / RHeff are contracted on first use only: the split matvec needs neither
    assert H._LHeff is None and H._RHeff is None
    assert H.LHeff.get_leg_labels() == ['(vR*.p0)', 'wR', '(vR.p0*)'] and H._RHeff is None
    # the two reshapes of theta are views now: only the transpositions inside the three contractions are left
    view_th = theta.split_legs(['(vL.p0)', '(p1.vR)'], _view=True)
    assert view_th._buf.data_ptr() == theta._buf.data_ptr()
    assert theta.split_legs(['(vL.p0)', '(p1.vR)'])._buf.data_ptr() != theta._buf.data_ptr()
    assert n_copies <= 4
    # with charges the reshapes move blocks: never a view
    M = SpinChain({'L': 8, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
    psi = MPS.from_product_state(M.lat_sites, ['up', 'down'] * 4)
    eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': True, 'combine': True, 'trunc_params': {'chi_max': 16, 'svd_min': 1e-12}})
    eng.sweep()
    H = TwoSiteH(eng.env, 3, combine=True, matvec_order='split')
    theta = H.combine_theta(psi.get_theta(3, 2))
    if theta.stored_blocks > 1:
        assert theta.split_legs(['(vL.p0)', '(p1.vR)'], _view=True)._buf.data_ptr() != theta._buf.data_ptr()


def test_matvec_identity_env_routes(fake_device):
    """split-order matvec with `identity_env=True`: the identity components LP[IdL], RP[IdR] of the environments are
    skipped (D-1 instead of D large GEMMs per side); same result on canonical states (dense, U(1), U(1)xU(1), and dense
    with K1 + K2 = D d^2 = 96 > 32, where W0 W1 is applied by npc.tensordot); falls back when the environment component is
    not the identity"""
    from tenpy_b200.models import TFIChain, SpinChain, FermiHubbardChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    cases = [(TFIChain({'L': 8, 'J': 1., 'g': 1.1, 'conserve': None}), ['up'] * 8, None),
             (SpinChain({'L': 8, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'conserve': 'Sz'}), ['up', 'down'] * 4, True),
             (FermiHubbardChain({'L': 6, 't': 1., 'U': 4., 'mu': 0.}), ['up', 'down'] * 3, True),
             (FermiHubbardChain({'L': 6, 't': 1., 'U': 4., 'mu': 0., 'cons_N': None, 'cons_Sz': None}), ['up', 'down'] * 3,
              None)]
    for M, state, mixer in cases:
        psi = MPS.from_product_state(M.lat_sites, state)
        eng = dmrg.TwoSiteDMRGEngine(psi, M, {'mixer': mixer, 'combine': True, 'matvec_order': 'combined',
                                              'trunc_params': {'chi_max': 24, 'svd_min': 1e-12}})
        eng.sweep()
        eng.sweep()
        eng.mixer_cleanup()
        psi.canonical_form()
        eng.env.clear()
        used = 0
        for i0 in range(psi.L - 1):
            Hc = TwoSiteH(eng.env, i0, combine=True, matvec_order='combined')
            Hi = TwoSiteH(eng.env, i0, combine=True, matvec_order='split')
            Hi.identity_env = True
            theta = Hc.combine_theta(psi.get_theta(i0, 2))
            a, b = Hc.matvec(theta), Hi.matvec(theta)
            if mixer is None and Hi._id_env:      # no charges: the two components of t2 are shared views, nothing is gathered
                n_take = fake_device.calls.get('take_blocks', 0)
                c = Hi.matvec(theta)     # TFI: the replayed kernel sequence; dense Hubbard (K1 + K2 > 32): W0 W1 by tensordot
                assert fake_device.calls.get('take_blocks', 0) == n_take
                assert npc.norm(c - b) <= 1e-14 * max(npc.norm(b), 1e-300)
            used += int(bool(Hi._id_env))
            assert a.get_leg_labels() == b.get_leg_labels()
            assert npc.norm(a - b) <= 1e-11 * max(npc.norm(a), 1e-300), (i0, npc.norm(a - b), npc.norm(a))
        assert used >= psi.L - 3            # the boundary bonds may have 1-dimensional MPO legs
    # dense case with the fused two-segment kernel (b200_mid_contract2_f64)
    M0, state0, _ = cases[0]
    psi0 = MPS.from_product_state(M0.lat_sites, state0)
    eng0 = dmrg.TwoSiteDMRGEngine(psi0, M0, {'mixer': None, 'combine': True, 'trunc_params': {'chi_max': 24, 'svd_min': 1e-12}})
    eng0.sweep()
    eng0.sweep()
    psi0.canonical_form()
    eng0.env.clear()
    for i0 in range(1, psi0.L - 2):
        Hc = TwoSiteH(eng0.env, i0, combine=True, matvec_order='combined')
        Hf = TwoSiteH(eng0.env, i0, combine=True, matvec_order='split')
        Hf.identity_env = True
        theta = Hc.combine_theta(psi0.get_theta(i0, 2))
        n0 = fake_device.calls.get('mid_contract2', 0)
        a, b = Hc.matvec(theta), Hf.matvec(theta)
        assert fake_device.calls.get('mid_contract2', 0) == n0 + 1
        assert npc.norm(a - b) <= 1e-11 * max(npc.norm(a), 1e-300)
        # second call on the same bond: the recorded raw kernel sequence is replayed (no Array-level bookkeeping)
        assert Hf._dense_recipe is not None
        n_plan = fake_device.calls.get('tdot_plan', 0)
        c = Hf.matvec(theta)
        assert fake_device.calls.get('mid_contract2', 0) == n0 + 2 and fake_device.calls.get('tdot_plan', 0) == n_plan
        assert c.get_leg_labels() == b.get_leg_labels() and c._layout is b._layout
        assert npc.norm(c - b) <= 1e-14 * max(npc.norm(b), 1e-300)
        c2 = Hf.matvec(theta * 2.)
        assert npc.norm(c2 - 2. * b) <= 1e-13 * max(npc.norm(b), 1e-300)
    # not applicable: an environment whose IdL component is not the identity -> the plain split order, same result
    H = TwoSiteH(eng.env, 2, combine=True, matvec_order='split')
    H.identity_env = True
    H.LP = H.LP * 1.5
    Href = TwoSiteH(eng.env, 2, combine=True, matvec_order='split')
    Href.LP = Href.LP * 1.5
    theta = H.combine_theta(psi.get_theta(2, 2))
    assert npc.norm(H.matvec(theta) - Href.matvec(theta)) < 1e-13 * npc.norm(Href.matvec(theta)) and H._id_env is False
    # whole runs with the option
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    res, psi = _run_dmrg(M, ['up'] * 20, {'mixer': None, 'max_E_err': 1e-10, 'combine': True, 'matvec_order': 'split',
                                         'identity_env': True, 'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['tfi_S'])) < 1e-8
    L = 16
    M = SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
    opts = {'mixer': True, 'mixer_params': {'amplitude': 1e-5, 'decay': 2., 'disable_after': 6}, 'max_E_err': 1e-11,
            'max_S_err': 1e-8, 'trunc_params': {'chi_max': 60, 'svd_min': 1e-10}, 'combine': True, 'max_sweeps': 20,
            'matvec_order': 'split', 'identity_env': True}
    res, psi = _run_dmrg(M, ['up', 'down'] * (L // 2), opts)
    assert abs(res['E'] - g['xxz_E']) < 1e-10 * abs(g['xxz_E'])


def test_identity_env_deferred_check_rejects(fake_device):
    """The engine defers the numerical test of the identity-environment shortcut to the first read-back of its Lanczos
    iteration; on a state that is NOT in canonical form the test fails, the iteration restarts with the plain contraction
    order and the run gives the same result as with the shortcut switched off."""
    from tenpy_b200.models import TFIChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    L = 10
    M = TFIChain({'L': L, 'J': 1., 'g': 1.3, 'conserve': None})
    res = {}
    for ident in (True, False):
        psi = MPS.from_product_state(M.lat_sites, ['up'] * L)
        psi._B[6] = psi._B[6] * 1.7          # breaks the right-canonical form: RP[IdR] = 1.7^2 left of site 6
        rej0 = TwoSiteH.stats['identity_env_rejected']
        out = dmrg.run(psi, M, {'mixer': None, 'max_E_err': 1e-11, 'combine': True, 'matvec_order': 'split',
                                'diag_method': 'lanczos', 'identity_env': ident,
                                'trunc_params': {'chi_max': 20, 'svd_min': 1e-10}})
        res[ident] = (out['E'], TwoSiteH.stats['identity_env_rejected'] - rej0)
    assert res[True][1] >= 1                      # the deferred test fired at least once ...
    assert abs(res[True][0] - res[False][0]) < 1e-10 * abs(res[False][0])      # ... and the result is unaffected
