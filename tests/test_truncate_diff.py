"""`tenpy_b200.linalg.truncation.truncate` (own formulation: conditions on the number of kept values) against the
reference's `truncate` (truncation.py:146) on randomised spectra and option combinations: same number of kept values, same
norm, same truncation error.  The reference's results for these seeded inputs are stored in tests/golden/truncate.npz
(tests/golden/make_golden_truncate.py)."""
import warnings

import numpy as np

import helpers as h


def test_truncate_matches_reference_randomised():
    from tenpy_b200.linalg.truncation import truncate as mine
    g = h.load('truncate.npz')
    rng = np.random.default_rng(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
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
            assert len(S) == g['n'][trial], trial       # the inputs are the ones the reference saw
            m1, n1, e1 = mine(S, dict(opts))
            m2, n2, e2 = g['kept'][trial], g['norm'][trial], g['eps'][trial]
            assert m1.sum() == m2 and abs(n1 - n2) < 1e-14 and abs(e1.eps - e2) < 1e-14, (opts, S)
