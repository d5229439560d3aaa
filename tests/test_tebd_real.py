"""Real-time TEBD (``exp(-i dt H)``) of the UNMODIFIED reference ``TEBDEngine`` on the tenpy_b200 engine (dropin), against
the numbers of the plain reference (tests/golden/tebd_real.npz, written by tests/golden/make_golden_tebd_real.py).

The cases run in a child process (tests/dropin/run_tebd_real.py): XXZ (Sz), TFI (no conservation) and Hubbard (N, Sz)
from product states at orders 2 and 4, and a dynamical correlation through ``apply_local_op(mid, 'Sp', unitary=False)``
and ``overlap``.  Only gauge-independent quantities are compared: bond energies, Sz, one correlation function, the norm
and the truncation error to 1e-9 absolute; entanglement entropies to 1e-8; bond dimensions exactly; the complex overlap to
1e-9 in modulus and phase."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, 'tests', 'dropin', 'run_tebd_real.py')


def _reference_available():
    sys.path.insert(0, ROOT)
    from tenpy_b200 import dropin
    return dropin.reference_path() is not None


def _run(mode):
    out = subprocess.run([sys.executable, RUNNER, mode], capture_output=True, text=True, timeout=1200, cwd='/tmp')
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def _check(got):
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'tebd_real.npz'))
    cases = sorted({k.rsplit('_', 1)[0] for k in gold.files})
    assert sorted(got) == cases
    for case in cases:
        rec = got[case]
        assert rec['chi'] == gold[case + '_chi'].tolist(), case
        np.testing.assert_allclose(rec['S'], gold[case + '_S'], rtol=0, atol=1e-8, err_msg=case)
        for key in ('Ebond', 'Sz', 'corr', 'norm', 'eps'):
            np.testing.assert_allclose(rec[key], gold[case + '_' + key], rtol=0, atol=1e-9, err_msg=case + ' ' + key)
        if case + '_overlap' in gold.files:
            ov, ref = complex(*rec['overlap']), complex(*gold[case + '_overlap'])
            assert abs(abs(ov) - abs(ref)) <= 1e-9, (ov, ref)
            assert abs(np.angle(ov / ref)) <= 1e-9, (ov, ref)


@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_real_time_tebd_host_logic():
    """the engine plumbing of complex states (CPU test double of the device library)"""
    _check(_run('fake'))


@pytest.mark.gpu
@pytest.mark.skipif(not _reference_available(), reason='reference package not available')
def test_real_time_tebd_gpu(gpu_lib):
    """the same on the H100: complex block-Jacobi SVD and complex Householder QR kernels"""
    _check(_run('cuda'))
