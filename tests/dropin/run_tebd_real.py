#!/usr/bin/env python
"""Real-time evolution ``exp(-i dt H)`` with the UNMODIFIED reference ``TEBDEngine`` running on the tenpy_b200 engine
(tenpy_b200.dropin): complex states, complex block SVD / QR, complex measurements.  Executed in its own process by
tests/test_tebd_real.py (the seeding has to happen before the first ``import tenpy``).

    python tests/dropin/run_tebd_real.py fake|cuda

Prints one JSON line: {case: {quantity: value}}.  Only gauge-independent quantities are recorded (the phases of the singular
vectors are arbitrary).  tests/golden/make_golden_tebd_real.py runs the same cases with the plain reference.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings('ignore')

DT = 0.05
N_STEPS = 8
TRUNC = {'chi_max': 128, 'svd_min': 1.e-10}


def _models():
    from tenpy.models.tf_ising import TFIChain
    from tenpy.models.spins import SpinChain
    from tenpy.models.hubbard import FermiHubbardChain
    L = 10
    yield 'xxz', SpinChain(dict(L=L, S=0.5, Jx=1., Jy=1., Jz=1.3, hz=0., bc_MPS='finite', conserve='Sz')), \
        ['up', 'down'] * (L // 2)
    yield 'tfi', TFIChain(dict(L=L, J=1., g=1.2, bc_MPS='finite', conserve=None)), ['up'] * L
    L = 6
    yield 'hub', FermiHubbardChain(dict(L=L, t=1., U=3., mu=0., bc_MPS='finite', cons_N='N', cons_Sz='Sz')), \
        ['up', 'down'] * (L // 2)


def _record(M, psi, eng):
    L = psi.L
    mid = L // 2
    return {'Ebond': [float(x) for x in np.real(M.bond_energies(psi))],
            'S': [float(x) for x in psi.entanglement_entropy()],
            'chi': [int(c) for c in psi.chi],
            'Sz': [float(x) for x in np.real(psi.expectation_value('Sz'))],
            'corr': [float(x) for x in np.real(psi.correlation_function('Sz', 'Sz', sites1=[mid - 1],
                                                                         sites2=list(range(L)))[0])],
            'norm': float(psi.norm),
            'eps': float(eng.trunc_err.eps)}


def run_cases():
    from tenpy.algorithms import tebd
    from tenpy.networks.mps import MPS
    out = {}
    for name, M, state in _models():
        sites = M.lat.mps_sites()
        for order in (2, 4):
            psi = MPS.from_product_state(sites, state, bc='finite')
            eng = tebd.TEBDEngine(psi, M, {'order': order, 'dt': DT, 'N_steps': N_STEPS, 'trunc_params': TRUNC})
            eng.run()
            out['{0}_o{1}'.format(name, order)] = _record(M, psi, eng)
    # dynamical correlation <neel(t)| S^-_{mid-1} e^{-iHt} S^+_mid |neel> (S^+ is not unitary: apply_local_op brings the
    # complex state back to canonical form, i.e. complex QR and SVD)
    name, M, state = next(_models())
    sites = M.lat.mps_sites()
    L = len(sites)
    psi = MPS.from_product_state(sites, state, bc='finite')
    phi = psi.copy()
    phi.apply_local_op(L // 2, 'Sp', unitary=False)
    for st in (psi, phi):
        eng = tebd.TEBDEngine(st, M, {'order': 2, 'dt': DT, 'N_steps': N_STEPS, 'trunc_params': TRUNC})
        eng.run()
    chi = psi.copy()
    chi.apply_local_op(L // 2 - 1, 'Sp', unitary=False)
    ov = complex(chi.overlap(phi))
    rec = _record(M, phi, eng)
    rec['overlap'] = [ov.real, ov.imag]
    out['xxz_dyn'] = rec
    return out


def main(mode):
    from run_reference_drivers import setup
    setup(mode)
    if mode == 'fake':       # the numpy test double with the complex decompositions (tests/fake_device_complex.py)
        from tenpy_b200 import backend
        from fake_device_complex import FakeComplexDeviceLib
        backend.use_library(FakeComplexDeviceLib())
    print(json.dumps(run_cases()))


if __name__ == '__main__':
    main(sys.argv[1])
