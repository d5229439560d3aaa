"""Lanczos on complex vectors: the ground state of a random complex Hermitian block-sparse operator against dense numpy,
through the device-scalar route (both planes of a Krylov vector in one buffer, one dot launch per iteration) and through
the host-scalar loop, on the CPU test double (tests/fake_device.py) and on the GPU."""
import numpy as np
import pytest


@pytest.fixture
def fake_device_eigh_z(fake_device):
    return fake_device


class _Op:
    """H acting on the first leg of a two-leg vector (the second leg a spectator); counts its matvecs"""

    def __init__(self, H):
        self.H, self.n = H, 0

    def matvec(self, v):
        self.n += 1
        from tenpy_b200.linalg import np_conserved as npc
        return npc.tensordot(self.H, v, axes=('p*', 'p'))


def _problem(seed):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(seed)
    ci = npc.ChargeInfo([1], ['N'])
    lp = npc.LegCharge.from_qind(ci, [0, 9, 22, 30, 41], [[-1], [0], [1], [2]], +1)
    ls = npc.LegCharge.from_qind(ci, [0, 2, 5, 6], [[-1], [0], [1]], +1)
    qp, qs = lp.to_qflat()[:, 0], ls.to_qflat()[:, 0]
    n = lp.ind_len
    x = rng.standard_normal((n, n)) + 1.j * rng.standard_normal((n, n))
    h = (x + x.conj().T) * np.equal.outer(qp, qp)
    H = npc.ComplexArray.from_ndarray(h, [lp, lp.conj()], labels=['p', 'p*'])
    allowed = np.add.outer(qp, qs) == 0                  # qtotal 0 of the vector
    v = (rng.standard_normal(allowed.shape) + 1.j * rng.standard_normal(allowed.shape)) * allowed
    psi = npc.ComplexArray.from_ndarray(v, [lp, ls], labels=['p', 's'])
    big = np.kron(h, np.eye(ls.ind_len))
    idx = np.nonzero(allowed.reshape(-1))[0]
    E0 = np.linalg.eigvalsh(big[np.ix_(idx, idx)])[0]
    return H, psi, E0, h


def _lanczos_case(lib, device_scalars):
    from tenpy_b200.linalg import krylov_based, np_conserved as npc
    H, psi, E0, h = _problem(5)
    calls = {'dot': 0}
    real_dot = lib.dot

    def counting_dot(*args):
        calls['dot'] += 1
        return real_dot(*args)
    lib.dot = counting_dot
    try:
        op = _Op(H)
        opts = {'N_min': 2, 'N_max': 60, 'P_tol': 1e-30, 'E_tol': 1e-15, 'min_gap': 1e-12,
                'device_scalars': device_scalars}
        E, psi_f, N = krylov_based.LanczosGroundState(op, psi, opts).run()
    finally:
        del lib.dot                                  # the class's method again
    assert abs(E - E0) <= 1e-12 * abs(E0), (E, E0)
    assert isinstance(psi_f, npc.ComplexArray)
    v = psi_f.to_ndarray()
    assert abs(np.linalg.norm(v) - 1.) <= 1e-12
    hv = np.tensordot(h, v, axes=(1, 0))
    assert np.linalg.norm(hv - E0 * v) <= 1e-6 * abs(E0)
    if device_scalars:
        # device-scalar route: one dot per iteration, the start norm and the result norm; no host fallback
        assert calls['dot'] == N + 2, (calls['dot'], N)
        assert op.n == N
    return E


def test_complex_lanczos_fake(fake_device_eigh_z):
    E_dev = _lanczos_case(fake_device_eigh_z, True)
    E_host = _lanczos_case(fake_device_eigh_z, False)
    assert abs(E_dev - E_host) <= 1e-12 * abs(E_dev)


@pytest.mark.gpu
def test_complex_lanczos_gpu(gpu_lib):
    E_dev = _lanczos_case(gpu_lib, True)
    E_host = _lanczos_case(gpu_lib, False)
    assert abs(E_dev - E_host) <= 1e-12 * abs(E_dev)
