#!/usr/bin/env python
"""Golden results of the reference's `truncate` (tenpy/linalg/truncation.py) on the seeded spectra and options of
tests/test_truncate_diff.py (the same generator), generated with the UNMODIFIED reference:

    TENPY_NO_CYTHON=1 TENPY_REFERENCE=<tenpy checkout> python tests/golden/make_golden_truncate.py

Per trial: length of the spectrum (to check that the test regenerates the same inputs), number of kept values, norm of
the kept part and truncation error."""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
os.environ.setdefault('TENPY_NO_CYTHON', '1')
sys.path.insert(0, os.environ['TENPY_REFERENCE'])
warnings.simplefilter('ignore')
from tenpy.linalg.truncation import truncate  # noqa: E402
from tenpy.tools.params import Config  # noqa: E402

out = {k: [] for k in ('n', 'kept', 'norm', 'eps')}
rng = np.random.default_rng(0)
for trial in range(1500):
    n = int(rng.integers(1, 40))
    kind = rng.integers(0, 4)
    if kind == 0:
        S = rng.random(n)
    elif kind == 1:
        S = np.exp(-rng.random(n) * 40)
    elif kind == 2:
        S = np.repeat(rng.random(max(1, n // 3)), 3)[:n]
    else:
        S = np.concatenate([rng.random(n // 2 + 1), np.zeros(n // 2)])
    S = S / np.linalg.norm(S)
    opts = {}
    if rng.random() < .8:
        opts['chi_max'] = int(rng.integers(1, 45)) if rng.random() < .9 else None
    if rng.random() < .3:
        opts['chi_min'] = int(rng.integers(1, 45))
    if rng.random() < .3:
        opts['degeneracy_tol'] = float(10 ** rng.uniform(-8, -1))
    if rng.random() < .7:
        opts['svd_min'] = float(10 ** rng.uniform(-16, -1)) if rng.random() < .9 else None
    if rng.random() < .7:
        opts['trunc_cut'] = float(10 ** rng.uniform(-16, -0.5)) if rng.random() < .9 else None
    mask, norm, err = truncate(S, Config(dict(opts), 'trunc'))
    out['n'].append(len(S))
    out['kept'].append(int(mask.sum()))
    out['norm'].append(norm)
    out['eps'].append(err.eps)
np.savez_compressed(os.path.join(HERE, 'truncate.npz'), n=np.array(out['n'], dtype=np.int8),
                    kept=np.array(out['kept'], dtype=np.int8),
                    norm=np.array(out['norm']), eps=np.array(out['eps']))
print('trials', len(out['n']))
