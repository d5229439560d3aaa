#!/usr/bin/env python
"""Time one two-site TDVP sweep of the XXZ chain (Sz conserved, L = 32) at saturated bond dimension, in three arms:

* ``reference``: the reference's ``TwoSiteTDVPEngine`` on the drop-in (its own LanczosEvolution and TwoSiteH);
* ``fast``:      ``dropin.fast_tdvp_engine()`` (the engine's LanczosEvolution and split-order matvec in the reference engine);
* ``engine``:    the engine's own ``tenpy_b200.algorithms.tdvp.TwoSiteTDVPEngine``.

    python profiles/tdvp_bench.py [--chis 128 256 512] [--dry-run]

The state is prepared by a few DMRG sweeps at ``chi_max = chi`` followed by two untimed TDVP sweeps (so that every inner
bond carries chi states), then one TDVP sweep is timed (CUDA-synchronised wall clock).  For each arm it prints one JSON
line with the sweep seconds, the matvecs per bond update and the host read-backs (device-to-host copies) of the sweep,
next to the name and power limit of the GPU.  ``--dry-run`` runs every arm at L = 8, chi = 8 on the CPU test double of
the device library (tests/fake_device.py): the numbers then check the plumbing only, the times mean nothing.  Each arm
runs in its own process (the drop-in has to be installed before the first ``import tenpy``).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def _gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'not measured (no GPU)'
    except (OSError, subprocess.SubprocessError):
        return 'not measured (no GPU)'


class _Counters:
    """host read-backs and matvecs, counted on the CPU by wrapping the few functions that do them"""

    def __init__(self):
        import torch
        from tenpy_b200 import backend
        self.readbacks = 0
        self.matvecs = 0
        counters = self
        for name in ('to_host', 'read_scalar'):
            fn = getattr(backend, name)

            def wrapped(*a, _fn=fn, **k):
                counters.readbacks += 1
                return _fn(*a, **k)
            setattr(backend, name, wrapped)
        self.torch = torch

    def wrap_matvec(self, cls):
        counters = self
        orig = cls.matvec

        def matvec(self, theta):
            counters.matvecs += 1
            return orig(self, theta)
        cls.matvec = matvec


def _setup(dry):
    from tenpy_b200 import backend
    if dry:
        from fake_device import FakeDeviceLib
        import fake_krylov_combine
        import fake_mid_contract_z
        backend.use_library(fake_mid_contract_z.install(fake_krylov_combine.install(FakeDeviceLib())))
    else:
        from tenpy_b200._lib import DeviceLib
        backend.use_library(DeviceLib())
    return backend.get_lib()


def run_arm(arm, chi, L, dry):
    lib = _setup(dry)
    opts_dmrg = {'mixer': True, 'max_sweeps': 4, 'min_sweeps': 4, 'trunc_params': {'chi_max': chi, 'svd_min': 0.},
                 'combine': True}
    tdvp_opts = {'dt': 0.05, 'N_steps': 1, 'trunc_params': {'chi_max': chi, 'svd_min': 0.}}
    if arm == 'engine':
        from tenpy_b200.algorithms import dmrg, tdvp
        from tenpy_b200.algorithms import mps_common
        from tenpy_b200.models import SpinChain
        from tenpy_b200.networks.mps import MPS
        M = SpinChain({'L': L, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'conserve': 'Sz'})
        psi = MPS.from_product_state(M.lat_sites, ['up', 'down'] * (L // 2))
        dmrg.run(psi, M, opts_dmrg)
        eng = tdvp.TwoSiteTDVPEngine(psi, M, tdvp_opts)
        Hcls = [mps_common.TwoSiteH, mps_common.OneSiteH]
    else:
        from tenpy_b200 import dropin
        dropin.install()
        from tenpy.algorithms import dmrg, tdvp, mps_common
        from tenpy.models.spins import SpinChain
        from tenpy.networks.mps import MPS
        M = SpinChain({'L': L, 'S': 0.5, 'Jx': 1., 'Jy': 1., 'Jz': 1., 'bc_MPS': 'finite', 'conserve': 'Sz'})
        psi = MPS.from_product_state(M.lat.mps_sites(), ['up', 'down'] * (L // 2), bc='finite')
        dmrg.run(psi, M, opts_dmrg)
        Eng = tdvp.TwoSiteTDVPEngine if arm == 'reference' else dropin.fast_tdvp_engine()
        tdvp_opts['combine'] = False          # the reference's TDVP engines run with its default combine=False
        eng = Eng(psi, M, tdvp_opts)
        Hcls = [Eng.EffectiveH, mps_common.OneSiteH]
    eng.run()                                 # two untimed sweeps: bond dimensions saturate, plans and caches warm
    eng.run()
    cnt = _Counters()
    for c in Hcls:
        cnt.wrap_matvec(c)
    lib.synchronize()
    t0 = time.perf_counter()
    eng.run()
    lib.synchronize()
    sec = time.perf_counter() - t0
    n_updates = 2 * (L - 2) + 1
    return {'arm': arm, 'L': L, 'chi': chi, 'max_chi': int(max(psi.chi)), 'sweep_s': sec if not dry else None,
            'matvecs_per_bond': cnt.matvecs / n_updates, 'readbacks_per_sweep': cnt.readbacks,
            'gpu': 'not measured (CPU test double)' if dry else _gpu_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chis', type=int, nargs='*', default=[128, 256, 512])
    ap.add_argument('--arms', nargs='*', default=['reference', 'fast', 'engine'])
    ap.add_argument('--L', type=int, default=32)
    ap.add_argument('--dry-run', action='store_true')
    ap.add_argument('--one', nargs=2, metavar=('ARM', 'CHI'), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one:
        print(json.dumps(run_arm(a.one[0], int(a.one[1]), a.L, a.dry_run)))
        return
    chis, L = ([8], 8) if a.dry_run else (a.chis, a.L)
    for chi in chis:
        for arm in a.arms:
            cmd = [sys.executable, os.path.abspath(__file__), '--one', arm, str(chi), '--L', str(L)] + \
                (['--dry-run'] if a.dry_run else [])
            out = subprocess.run(cmd, capture_output=True, text=True)
            if out.returncode != 0:
                print(json.dumps({'arm': arm, 'chi': chi, 'error': out.stderr.strip().splitlines()[-1:]}))
            else:
                print(out.stdout.strip().splitlines()[-1], flush=True)


if __name__ == '__main__':
    main()
