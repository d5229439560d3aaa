"""dev probe (not a test): effective-H matvec at a saturated centre bond, reference order (LHeff.theta.RHeff,
4 D d^3 chi^3 flop) against the 'split' order (LP, W0 W1, RP on the split theta, 4 D d^2 chi^3 flop; W0 W1 applied by the
streaming kernel b200_mid_contract(2)_f64 on these dense shapes).

    python tests/dev_matvec_order_probe.py [chi=1024] [L=24] [reps=10]

Prints one JSON line per order: ms per matvec (CUDA events), per kernel-family ms, relative difference of results.
"""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, '.')
from tenpy_b200 import backend


def main():
    chi = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    L = int(sys.argv[2]) if len(sys.argv) > 2 else 24
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    lib = backend.get_lib()
    import bench
    from tenpy_b200.models import TFIChain
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.algorithms.mps_common import TwoSiteH
    from tenpy_b200.linalg import np_conserved as npc
    model = TFIChain({'L': L, 'J': 1., 'g': 1., 'conserve': None})
    psi = bench.synthetic_mps(model, L, chi, 2, seed=0)
    eng = dmrg.TwoSiteDMRGEngine(psi, model, {'mixer': None, 'combine': True,
                                              'trunc_params': {'chi_max': chi, 'svd_min': 1e-45}})
    i0 = L // 2 - 1
    eng.env.get_LP(i0, store=True)
    eng.env.get_RP(i0 + 1, store=True)
    cuda = lib.device.type == 'cuda'
    out = {}
    for order in ('combined', 'split'):
        H = TwoSiteH(eng.env, i0, combine=True, matvec_order=order)
        theta = H.combine_theta(psi.get_theta(i0, 2))
        for _ in range(3):
            res = H.matvec(theta)
        lib.synchronize()
        if cuda:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        t0 = time.perf_counter()
        for _ in range(reps):
            res = H.matvec(theta)
        if cuda:
            ev1.record()
        lib.synchronize()
        wall = (time.perf_counter() - t0) / reps * 1e3
        ms = ev0.elapsed_time(ev1) / reps if cuda else wall
        lib.profile = {}
        for _ in range(reps):
            H.matvec(theta)
        fam = {k: round(v[1] / reps, 4) for k, v in lib.profile_summary().items()} if cuda else {}
        lib.profile = None
        out[order] = res
        d, D = 2, 3
        print(json.dumps({'order': order, 'chi': chi, 'theta_shape': list(theta.shape), 'ms_per_matvec': round(ms, 4),
                          'wall_ms': round(wall, 4), 'family_ms': fam,
                          'reference_equivalent_tflops': 4. * D * d**3 * chi**3 / (ms * 1e-3) / 1e12}))
    diff = npc.norm(out['combined'] - out['split']) / npc.norm(out['combined'])
    print(json.dumps({'rel_diff_split_vs_combined': diff}))
    assert diff < 1e-12


if __name__ == '__main__':
    main()
