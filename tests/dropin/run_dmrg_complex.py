#!/usr/bin/env python
"""Ground-state DMRG of a complex Hamiltonian with the UNMODIFIED reference drivers on the tenpy_b200 engine
(tenpy_b200.dropin): the reference's ``FermionicHaldaneModel`` (complex next-nearest-neighbour hoppings) on a 2 x 3
cylinder, run through the reference's ``TwoSiteDMRGEngine`` and through ``dropin.fast_two_site_engine()``.  Executed in its
own process by tests/test_dmrg_complex_dropin.py (the seeding has to happen before the first ``import tenpy``).

    python tests/dropin/run_dmrg_complex.py fake|cuda

Prints one JSON line: {engine: {'E', 'S', 'chi'}}.  tests/golden/make_golden_dmrg_complex.py runs the same case with the
plain reference.
"""
import json
import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings('ignore')

MODEL = dict(Lx=2, Ly=3, bc_MPS='finite', bc_y='cylinder', conserve='N', V=0.5)
DMRG = {'mixer': True, 'max_E_err': 1.e-12, 'max_S_err': 1.e-9, 'min_sweeps': 4, 'max_sweeps': 30, 'combine': True,
        'trunc_params': {'chi_max': 64, 'svd_min': 1.e-12}}


def run_case(Engine=None):
    """one DMRG run from the half-filled product state; `Engine`: an engine class (default: the reference's)"""
    import numpy as np
    from tenpy.algorithms import dmrg
    from tenpy.models.haldane import FermionicHaldaneModel
    from tenpy.networks.mps import MPS
    M = FermionicHaldaneModel(dict(MODEL))
    L = M.lat.N_sites
    psi = MPS.from_product_state(M.lat.mps_sites(), ['full', 'empty'] * (L // 2), bc='finite')
    eng = (Engine or dmrg.TwoSiteDMRGEngine)(psi, M, dict(DMRG))
    E, _ = eng.run()
    return {'E': float(np.real(E)), 'S': [float(s) for s in psi.entanglement_entropy()],
            'chi': [int(c) for c in psi.chi], 'H_dtype': str(np.dtype(M.H_MPO.dtype)),
            'psi_dtype': str(np.dtype(psi.dtype))}


def main(mode):
    from run_reference_drivers import setup
    dropin = setup(mode)
    if mode == 'fake':       # the numpy test double with the complex decompositions and the complex eigh
        from tenpy_b200 import backend
        from fake_device_eigh_z import FakeEighZDeviceLib
        lib = backend.use_library(FakeEighZDeviceLib())
    else:
        from tenpy_b200 import backend
        lib = backend.get_lib()
    out = {'reference_engine': run_case(), 'fast_engine': run_case(dropin.fast_two_site_engine())}
    if mode == 'fake':
        out['eigh_z_calls'] = lib.calls.get('block_eigh_z', 0)
    print(json.dumps(out))


if __name__ == '__main__':
    main(sys.argv[1])
