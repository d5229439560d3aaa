"""Ground-state DMRG of a complex Hamiltonian with the UNMODIFIED reference drivers on the tenpy_b200 engine (dropin): the
reference's ``FermionicHaldaneModel`` (complex next-nearest-neighbour hoppings; Lx = 2, Ly = 3 cylinder, N conserved,
V = 0.5, mixer on, chi_max = 64) through the reference's ``TwoSiteDMRGEngine`` and through
``dropin.fast_two_site_engine()``, against the plain reference (tests/golden/dmrg_complex.npz, written by
tests/golden/make_golden_dmrg_complex.py, which also stores the exact energy of the N = 6 sector from a dense
diagonalisation).

The case runs in a child process (tests/dropin/run_dmrg_complex.py).  E to 1e-10 (golden and exact), entanglement
entropies to 1e-8; the bond dimensions exactly, since chi_max = 64 = 2^(L/2) leaves every bond at its Hilbert-space
dimension."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, 'tests', 'dropin', 'run_dmrg_complex.py')


def _reference_available():
    sys.path.insert(0, ROOT)
    from tenpy_b200 import dropin
    return dropin.reference_path() is not None


def _run(mode):
    out = subprocess.run([sys.executable, RUNNER, mode], capture_output=True, text=True, timeout=1800, cwd='/tmp')
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def _check(got):
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'dmrg_complex.npz'))
    L = len(gold['chi']) + 1
    assert int(gold['sector_dim']) == 924
    assert gold['chi'].tolist() == [min(2**i, 2**(L - i)) for i in range(1, L)]
    for engine in ('reference_engine', 'fast_engine'):
        rec = got[engine]
        assert rec['H_dtype'] == 'complex128' and rec['psi_dtype'] == 'complex128', engine
        E = rec['E']
        assert abs(E - float(gold['E'])) <= 1e-10 * abs(float(gold['E'])), (engine, E, float(gold['E']))
        assert abs(E - float(gold['E_exact'])) <= 1e-10 * abs(float(gold['E_exact'])), (engine, E)
        np.testing.assert_allclose(rec['S'], gold['S'], rtol=0, atol=1e-8, err_msg=engine)
        assert rec['chi'] == gold['chi'].tolist(), engine


@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_complex_dmrg_dropin_host_logic():
    """the engine plumbing of complex Hamiltonians (CPU test double of the device library); the mixer diagonalises complex
    density matrices with the complex eigh"""
    got = _run('fake')
    _check(got)
    assert got['eigh_z_calls'] > 0


@pytest.mark.gpu
@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_complex_dmrg_dropin_gpu(gpu_lib):
    """the same on the H100: complex block eigh, SVD and Lanczos on the device"""
    _check(_run('cuda'))
