"""Ground-state DMRG of complex Hamiltonians on the engine's own driver (two-site engine, `models.SpinChain` with a
Dzyaloshinskii-Moriya term `D`), on the CPU test double (tests/fake_device.py) at small L and on the GPU larger.

* Gauge test: with ``Jx = Jy = J`` the DM term only twists the XY coupling, ``(J + iD)/2 S+_i S-_{i+1} + h.c.``; on an
  open chain ``prod_j exp(-i j phi Sz_j)`` removes the phase, so the chain is equivalent to the real XXZ chain with
  ``Jxx = sqrt(J^2 + D^2)``: the same energy, the same Schmidt values on every bond.
* Free fermions: at ``Jz = 0`` the Jordan-Wigner transformation gives a hopping chain with the exact energy of its filled
  single-particle levels (``Sz = 0``: ``L/2`` fermions).
* A case no gauge makes real (``Jx != Jy``, parity conserved) against a dense diagonalisation built here.
"""
import numpy as np
import pytest


@pytest.fixture
def fake_device_eigh_z(fake_device):
    return fake_device


MIXER_PARAMS = {'amplitude': 1e-5, 'decay': 2., 'disable_after': 6}


def _run(params, p_state, chi, mixer):
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    M = SpinChain(params)
    psi = MPS.from_product_state(M.lat_sites, p_state)
    opts = {'mixer': mixer, 'mixer_params': dict(MIXER_PARAMS), 'max_E_err': 1e-12, 'max_S_err': 1e-9,
            'min_sweeps': 4, 'max_sweeps': 30, 'combine': True,
            'trunc_params': {'chi_max': chi, 'svd_min': 1e-12}, 'lanczos_params': {'N_max': 40, 'P_tol': 1e-16}}
    res = dmrg.run(psi, M, opts)
    return M, psi, res['E']


def _chi_fixed(psi, chi_max):
    """bonds whose bond dimension chi_max or the Hilbert space fixes: chi = chi_max, or chi = d^min(i, L-i)"""
    L = psi.L
    full = [min(2**i, 2**(L - i)) for i in range(1, L)]
    return [j for j, (c, f) in enumerate(zip(psi.chi, full)) if c == chi_max or c == f]


def _gauge_case(L, chi, mixer):
    J, D, Jz, hz = 1., 0.6, 0.7, 0.1
    neel = ['up', 'down'] * (L // 2)
    Mc, psi_c, E_c = _run({'L': L, 'Jx': J, 'Jy': J, 'Jz': Jz, 'D': D, 'hz': hz, 'conserve': 'Sz'}, neel, chi, mixer)
    Mr, psi_r, E_r = _run({'L': L, 'Jx': np.hypot(J, D), 'Jy': np.hypot(J, D), 'Jz': Jz, 'hz': hz, 'conserve': 'Sz'},
                          neel, chi, mixer)
    assert Mc.H_MPO.dtype is np.complex128 and Mr.H_MPO.dtype is np.float64
    assert psi_c.dtype is np.complex128 and psi_r.dtype is np.float64
    assert abs(E_c - E_r) <= 1e-10 * abs(E_r), (E_c, E_r)
    S_c, S_r = psi_c.entanglement_entropy(), psi_r.entanglement_entropy()
    assert np.max(np.abs(S_c - S_r)) <= 1e-8, np.max(np.abs(S_c - S_r))
    fixed = _chi_fixed(psi_r, chi)
    assert len(fixed) > 0
    for j in fixed:
        assert psi_c.chi[j] == psi_r.chi[j], (j, psi_c.chi, psi_r.chi)
    assert np.max(psi_c.isometry_test()) < 1e-12


def _free_fermion_case(L, chi):
    J, D, hz = 1., 0.6, 0.1
    neel = ['up', 'down'] * (L // 2)
    _, psi, E = _run({'L': L, 'Jx': J, 'Jy': J, 'Jz': 0., 'D': D, 'hz': hz, 'conserve': 'Sz'}, neel, chi, False)
    # S+_i S-_{i+1} = c+_i c_{i+1}: hopping (J + iD)/2, -hz Sz = -hz (n - 1/2); Sz = 0 holds L/2 fermions
    h = np.diag(np.full(L - 1, (J + 1j * D) / 2.), 1)
    h = h + h.conj().T - hz * np.eye(L)
    E_exact = np.sum(np.linalg.eigvalsh(h)[:L // 2]) + hz * L / 2.
    assert abs(E - E_exact) <= 1e-10 * abs(E_exact), (E, E_exact)


def _dense_chain(L, Jx, Jy, Jz, D, hz):
    """the chain's Hamiltonian on all 2^L states (site 0 the most significant bit; bit 0 = up), scipy.sparse"""
    import scipy.sparse as sps
    sp = np.array([[0., 1.], [0., 0.]])
    sx = 0.5 * (sp + sp.T)
    sy = -0.5j * (sp - sp.T)
    sz = np.diag([0.5, -0.5])

    def op(o, i):
        return sps.kron(sps.kron(sps.identity(2**i), o), sps.identity(2**(L - i - 1)), format='csr')
    H = sps.csr_matrix((2**L, 2**L), dtype=np.complex128)
    for i in range(L - 1):
        H += Jx * op(sx, i) @ op(sx, i + 1) + Jy * op(sy, i) @ op(sy, i + 1) + Jz * op(sz, i) @ op(sz, i + 1)
        H += D * (op(sx, i) @ op(sy, i + 1) - op(sy, i) @ op(sx, i + 1))
    for i in range(L):
        H -= hz * op(sz, i)
    return H


def _parity_case(mixer):
    L, p = 12, {'Jx': 1.2, 'Jy': 0.8, 'Jz': 1., 'D': 0.5, 'hz': 0.3}
    _, psi, E = _run(dict(p, L=L, conserve='parity'), ['up'] * L, 64, mixer)
    H = _dense_chain(L, **p)
    n_up = L - np.array([bin(s).count('1') for s in range(2**L)])          # basis state bits: 0 = up, 1 = down
    idx = np.nonzero(n_up % 2 == L % 2)[0]                                    # the parity sector of all-up
    w, v = np.linalg.eigh(H[idx][:, idx].toarray())
    assert abs(E - w[0]) <= 1e-10 * abs(w[0]), (E, w[0])
    g = np.zeros(2**L, dtype=np.complex128)
    g[idx] = v[:, 0]
    s = np.linalg.svd(g.reshape(2**(L // 2), -1), compute_uv=False)
    s2 = s[s > 1e-15]**2
    S_mid = -np.sum(s2 * np.log(s2))
    assert abs(psi.entanglement_entropy()[L // 2 - 1] - S_mid) <= 1e-8


@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_gauge_fake(fake_device_eigh_z, monkeypatch, mixer):
    from tenpy_b200.algorithms import mps_common
    calls = fake_device_eigh_z.calls
    in_mixer = []
    svd_from_rho = mps_common.DensityMatrixMixer.svd_from_rho

    def counting(self, engine, rho_L, rho_R, theta, qtotal_LR):
        n0 = calls.get('block_eigh_z', 0)
        out = svd_from_rho(self, engine, rho_L, rho_R, theta, qtotal_LR)
        in_mixer.append(calls.get('block_eigh_z', 0) - n0)
        return out
    monkeypatch.setattr(mps_common.DensityMatrixMixer, 'svd_from_rho', counting)
    _gauge_case(16, 48, mixer)
    # the density-matrix mixer diagonalises rho_L and rho_R of the complex state by the complex eigh (two calls per bond;
    # none in the real run)
    assert bool(in_mixer) == mixer
    assert all(d in (0, 2) for d in in_mixer) and (sum(in_mixer) > 0) == mixer


def test_dm_chain_free_fermions_fake(fake_device_eigh_z):
    _free_fermion_case(16, 64)


@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_parity_ed_fake(fake_device_eigh_z, mixer):
    _parity_case(mixer)


def test_dm_zero_is_the_real_mpo(fake_device_eigh_z):
    """D = 0 builds the same real MPO as a chain without the parameter"""
    from tenpy_b200.models import SpinChain
    from tenpy_b200.linalg import np_conserved as npc
    p = {'L': 4, 'Jx': 1., 'Jy': 1., 'Jz': 0.7, 'hz': 0.1, 'conserve': 'Sz'}
    a, b = SpinChain(p).H_MPO, SpinChain(dict(p, D=0.)).H_MPO
    assert b.dtype is np.float64
    for i in range(4):
        Wa, Wb = a.get_W(i), b.get_W(i)
        assert type(Wb) is npc.Array
        assert np.array_equal(Wa.to_ndarray(), Wb.to_ndarray())


@pytest.mark.gpu
@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_gauge_gpu(gpu_lib, mixer):
    _gauge_case(64, 128, mixer)


@pytest.mark.gpu
def test_dm_chain_free_fermions_gpu(gpu_lib):
    _free_fermion_case(32, 128)


@pytest.mark.gpu
@pytest.mark.parametrize('mixer', [False, True], ids=['no-mixer', 'mixer'])
def test_dm_chain_parity_ed_gpu(gpu_lib, mixer):
    _parity_case(mixer)
