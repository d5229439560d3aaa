#!/usr/bin/env python
"""Golden real-time TDVP numbers generated with the UNMODIFIED reference on its own NumPy engine (build container only):

    TENPY_NO_CYTHON=1 PYTHONPATH=/root/reference python tests/golden/make_golden_tdvp.py

Runs the cases of tests/dropin/run_tdvp.py (two-site TDVP with ``dt = 0.05`` from product states: XXZ (Sz) L = 10,
TFI without charges L = 10, Hubbard (N, Sz) L = 6 and SpinChainNNN2 (Sz) L = 10 for 8 steps, the complex
FermionicHaldaneModel on a 2 x 3 cylinder for 4 steps; single-site TDVP for 8 steps after 4 two-site steps on the XXZ
chain) and stores the gauge-independent results in tdvp.npz."""
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
from run_tdvp import CASES, run_case  # noqa: E402

out = {}
for case in CASES:
    rec = run_case(case)
    for key, val in rec.items():
        out[case + '_' + key] = np.asarray(val)
    print(case, 'chi', rec['chi'], 'norm', rec['norm'], 'E', rec['E'], 'amp', rec['amp'])
np.savez_compressed(os.path.join(HERE, 'tdvp.npz'), **out)
