#!/usr/bin/env python
"""Complex against real block SVD on the H100, and one real-time TEBD step:

    python profiles/complex_svd_bench.py [--chis 256,512,1024] [--reps 3] [--no-tebd]

For each theta structure (TFI without conservation: one dense 2chi x 2chi block; XXZ with Sz conservation: the same total
size cut into charge sectors of Gaussian weights) `npc.svd` is timed on a complex theta and on a real theta with the same
blocks and the same singular values (logspace(0, -12)); `ratio` = complex / real.  The arithmetic of the complex Jacobi
rounds is about 4x the real one.  Then the reference's TEBDEngine (through tenpy_b200.dropin) evolves an XXZ chain in real
time and one more order-2 step is timed.  Prints the card name and power limit first; every time is a median over
--reps calls, each ended by a device synchronisation."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # pragma: no cover
        return 'unknown ({0})'.format(e)


def sector_sizes(total, structure):
    if structure == 'tfi':
        return [total]
    nsec = 2 * int(np.sqrt(total) / 4) + 1
    w = np.exp(-0.5 * ((np.arange(nsec) - nsec // 2) / (nsec / 5.)) ** 2)
    s = np.maximum(1, np.round(total * w / w.sum())).astype(int)
    s[nsec // 2] += total - s.sum()
    return [int(x) for x in s]


def thetas(npc, rng, chi, structure):
    sizes = sector_sizes(2 * chi, structure)
    ci = npc.ChargeInfo([1], ['Sz'])
    slices = np.concatenate([[0], np.cumsum(sizes)])
    charges = [[2 * i] for i in range(len(sizes))]
    lL = npc.LegCharge.from_qind(ci, slices, charges, +1)
    lR = npc.LegCharge.from_qind(ci, slices, charges, -1)
    cblocks, rblocks = [], []
    for n in sizes:
        s = np.logspace(0, -12, n)
        u, _ = np.linalg.qr(rng.standard_normal((n, n)) + 1.j * rng.standard_normal((n, n)))
        v, _ = np.linalg.qr(rng.standard_normal((n, n)) + 1.j * rng.standard_normal((n, n)))
        cblocks.append((u * s) @ v.conj().T)
        ur, _ = np.linalg.qr(rng.standard_normal((n, n)))
        vr, _ = np.linalg.qr(rng.standard_normal((n, n)))
        rblocks.append((ur * s) @ vr.T)
    qd = [[i, i] for i in range(len(sizes))]
    c = npc.Array.from_blocks([lL, lR], qd, cblocks, None, ['L', 'R'])
    r = npc.Array.from_blocks([lL, lR], qd, rblocks, None, ['L', 'R'])
    assert isinstance(c, npc.ComplexArray) and not isinstance(r, npc.ComplexArray)
    return c, r, sizes


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def tebd_step(reps):
    """XXZ L=32 (Sz), Neel state, real time dt=0.05 order 2, chi_max 256: 30 steps to grow chi, then one step timed"""
    from tenpy_b200 import dropin
    if dropin.install() is None:
        return {'tebd': 'reference not available'}
    from tenpy.algorithms import tebd
    from tenpy.models.spins import SpinChain
    from tenpy.networks.mps import MPS
    L = 32
    M = SpinChain(dict(L=L, S=0.5, Jx=1., Jy=1., Jz=1., bc_MPS='finite', conserve='Sz'))
    psi = MPS.from_product_state(M.lat.mps_sites(), ['up', 'down'] * (L // 2), bc='finite')
    eng = tebd.TEBDEngine(psi, M, {'order': 2, 'dt': 0.05, 'N_steps': 30,
                                   'trunc_params': {'chi_max': 256, 'svd_min': 1e-10}})
    eng.run()
    eng.options['N_steps'] = 1
    t = timed(eng.run, reps)
    return {'tebd_L': L, 'tebd_chi_max_reached': int(max(psi.chi)), 'tebd_step_s': t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chis', default='256,512,1024')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--no-tebd', action='store_true')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('complex_svd_bench.py measures on the GPU; no CUDA device visible')
    print('card:', card())
    from tenpy_b200 import backend
    from tenpy_b200._lib import DeviceLib
    backend.use_library(DeviceLib())
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(0)
    for structure in ('tfi', 'xxz'):
        for chi in [int(c) for c in args.chis.split(',')]:
            c, r, sizes = thetas(npc, rng, chi, structure)
            npc.svd(c)
            npc.svd(r)   # warm-up of every shape
            tc = timed(lambda: npc.svd(c), args.reps)
            tr = timed(lambda: npc.svd(r), args.reps)
            print(json.dumps({'structure': structure, 'chi': chi, 'blocks': len(sizes), 'largest_block': max(sizes),
                              'complex_s': tc, 'real_s': tr, 'ratio': tc / tr}))
    if not args.no_tebd:
        print(json.dumps(tebd_step(args.reps)))


if __name__ == '__main__':
    main()
