#!/usr/bin/env python
"""Golden real-time TEBD numbers generated with the UNMODIFIED reference on its own NumPy engine (build container only):

    TENPY_NO_CYTHON=1 PYTHONPATH=/root/reference python tests/golden/make_golden_tebd_real.py

Runs the cases of tests/dropin/run_tebd_real.py (``TEBDEngine.run()`` with ``exp(-i dt H)`` for XXZ (Sz), TFI (no
conservation) and Hubbard (N, Sz) from product states at orders 2 and 4, and one dynamical correlation through
``apply_local_op(mid, 'Sp', unitary=False)``) and stores the gauge-independent results in tebd_real.npz."""
import os
import sys
import warnings

import numpy as np

os.environ.setdefault('TENPY_NO_CYTHON', '1')
sys.path.insert(0, os.environ.get('TENPY_REFERENCE', '/root/reference'))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'dropin'))
warnings.simplefilter('ignore')
import tenpy.linalg.np_conserved as npc  # noqa: E402
assert not npc.__name__.startswith('tenpy_b200'), 'must run with the plain reference'
from run_tebd_real import run_cases  # noqa: E402

out = {}
for case, rec in run_cases().items():
    for key, val in rec.items():
        out[case + '_' + key] = np.asarray(val)
    print(case, 'chi', rec['chi'], 'norm', rec['norm'], 'eps', rec['eps'], rec.get('overlap', ''))
np.savez_compressed(os.path.join(HERE, 'tebd_real.npz'), **out)
