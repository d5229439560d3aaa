#!/usr/bin/env python
"""Complex against real ground-state DMRG on the H100:

    python profiles/complex_dmrg_bench.py [--chis 256,512,1024] [--L 32] [--reps 3] [--conserve Sz,None] [--no-eigh]

1. One two-site sweep of the Dzyaloshinskii-Moriya chain (`SpinChain` Jx = Jy = 1, Jz = 0.7, D = 0.6, hz = 0.1, Sz
   conserved or no charges; complex MPO) against one sweep of the gauge-equivalent real XXZ chain (Jxx = sqrt(1 + D^2))
   from the same state: the real chain is run to chi, its MPS is carried over to the DM chain by the site-local gauge
   prod_j exp(-i j phi Sz_j) (exact: the same Schmidt values), then each arm does one warm-up sweep (environments) and
   one timed sweep at chi_max = chi (svd_min = 1e-45: the inner bonds stay at chi), no mixer.  Four arms, run one after
   the other in alternating order (--sweep-reps rounds): the complex chain with matvec_order='combined' (LHeff . theta .
   RHeff), the complex chain with 'auto' (the split order where the blocks are large), the complex chain with 'split' (the
   split order on every bond) and the real chain ('auto').
2. `npc.eigh` of a complex Hermitian against a real symmetric rho, one dense block of size chi, eigenvalues
   logspace(0, -12).

`ratio_*` = complex / real, `speedup` = combined / auto, `speedup_split` = combined / split.  Prints the card name and power limit first; every time is taken
around work that ends in a device synchronisation (a median over --reps for eigh, the minimum over the rounds for the
sweeps).  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

J, D, JZ, HZ = 1., 0.6, 0.7, 0.1


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # pragma: no cover
        return 'unknown ({0})'.format(e)


def synced(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def gauge(psi, M):
    """the MPS of the real chain carried over to the DM chain: B_j[vL, s, vR] * exp(-i j phi Sz_s), phi = atan2(D, J)"""
    from tenpy_b200.networks.mps import MPS
    phi = np.arctan2(D, J)
    Bs = []
    for j in range(psi.L):
        sz = np.real(np.diag(M.lat_sites[j].get_op('Sz').to_ndarray()))     # Sz in the (sorted) basis of the leg
        Bs.append(psi.get_B(j).astype(np.complex128).scale_axis(np.exp(-1j * j * phi * sz), 'p'))
    return MPS(M.lat_sites, Bs, [None if s is None else np.array(s) for s in psi._S], form=list(psi.form))


def sweep_times(L, chi, conserve, rounds):
    from tenpy_b200.algorithms import dmrg
    from tenpy_b200.models import SpinChain
    from tenpy_b200.networks.mps import MPS
    Mr = SpinChain({'L': L, 'Jx': np.hypot(J, D), 'Jy': np.hypot(J, D), 'Jz': JZ, 'hz': HZ, 'conserve': conserve})
    Mc = SpinChain({'L': L, 'Jx': J, 'Jy': J, 'Jz': JZ, 'D': D, 'hz': HZ, 'conserve': conserve})
    assert Mc.H_MPO.dtype is np.complex128
    psi = MPS.from_product_state(Mr.lat_sites, ['up', 'down'] * (L // 2))
    trunc = {'chi_max': chi, 'svd_min': 1e-45}      # (as bench.py: chi stays saturated, every sweep does the same work)
    ramp = {0: min(64, chi), 2: min(256, chi), 4: chi}
    dmrg.run(psi, Mr, {'mixer': None, 'combine': True, 'trunc_params': trunc, 'chi_list': ramp, 'min_sweeps': 6,
                       'max_sweeps': 6, 'max_E_err': 0.})
    res = {'chi': chi, 'conserve': str(conserve), 'max_chi_reached': int(max(psi.chi))}
    arms = [('complex_combined', Mc, 'combined'), ('complex_auto', Mc, 'auto'), ('complex_split', Mc, 'split'),
            ('real', Mr, 'auto')]
    times = {name: [] for name, _, _ in arms}
    for r in range(rounds):
        for name, M, order in (arms if r % 2 == 0 else arms[::-1]):
            state = MPS(Mr.lat_sites, [B.copy() for B in psi._B], list(psi._S), form=list(psi.form))
            if M is Mc:
                state = gauge(state, Mc)
            eng = dmrg.TwoSiteDMRGEngine(state, M, {'mixer': None, 'combine': True, 'trunc_params': trunc,
                                                    'matvec_order': order})
            eng.sweep()                                       # warm-up: environments, first launches of every shape
            t, _ = synced(eng.sweep)
            times[name].append(t)
            res['E_' + name] = float(eng.update_stats['E_total'][-1])
    for name in times:
        res['sweep_s_' + name] = min(times[name])
        res['all_s_' + name] = times[name]
    res['ratio_combined'] = res['sweep_s_complex_combined'] / res['sweep_s_real']
    res['ratio_auto'] = res['sweep_s_complex_auto'] / res['sweep_s_real']
    res['speedup'] = res['sweep_s_complex_combined'] / res['sweep_s_complex_auto']
    res['speedup_split'] = res['sweep_s_complex_combined'] / res['sweep_s_complex_split']
    res['dE_auto_combined'] = abs(res['E_complex_auto'] - res['E_complex_combined']) / abs(res['E_real'])
    return res


def eigh_times(chi, reps):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(chi)
    w = np.logspace(0, -12, chi)
    qc, _ = np.linalg.qr(rng.standard_normal((chi, chi)) + 1j * rng.standard_normal((chi, chi)))
    qr, _ = np.linalg.qr(rng.standard_normal((chi, chi)))
    leg = npc.LegCharge.from_trivial(chi)
    rc = npc.ComplexArray.from_ndarray((qc * w) @ qc.conj().T, [leg, leg.conj()], labels=['a', 'a*'])
    rr = npc.Array.from_ndarray((qr * w) @ qr.T, [leg, leg.conj()], labels=['a', 'a*'])
    res = {'n': chi}
    for name, rho in (('real', rr), ('complex', rc)):
        npc.eigh(rho)                                          # warm-up
        res['eigh_s_' + name] = float(np.median([synced(lambda: npc.eigh(rho))[0] for _ in range(reps)]))
    res['ratio'] = res['eigh_s_complex'] / res['eigh_s_real']
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chis', default='256,512,1024')
    ap.add_argument('--L', type=int, default=32)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--sweep-reps', type=int, default=2)
    ap.add_argument('--conserve', default='Sz')
    ap.add_argument('--no-eigh', action='store_true')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('complex_dmrg_bench.py measures on a CUDA device; none is visible')
    from tenpy_b200 import backend
    from tenpy_b200._lib import DeviceLib
    backend.use_library(DeviceLib())
    print(json.dumps({'card': card(), 'torch_device': torch.cuda.get_device_name(0)}), flush=True)
    chis = [int(c) for c in args.chis.split(',')]
    if not args.no_eigh:
        for chi in chis:
            print(json.dumps(dict(eigh_times(chi, args.reps), what='npc.eigh')), flush=True)
    for conserve in args.conserve.split(','):
        for chi in chis:
            res = sweep_times(args.L, chi, None if conserve == 'None' else conserve, args.sweep_reps)
            print(json.dumps(dict(res, what='two-site sweep', L=args.L)), flush=True)


if __name__ == '__main__':
    main()
