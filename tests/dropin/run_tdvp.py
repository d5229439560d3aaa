#!/usr/bin/env python
"""Real-time TDVP with the UNMODIFIED reference ``TwoSiteTDVPEngine`` / ``SingleSiteTDVPEngine`` on the tenpy_b200 engine
(tenpy_b200.dropin), and with ``dropin.fast_tdvp_engine()`` (the engine's Lanczos evolution and split-order matvec plugged
into the reference's engines).  Executed in its own process, one case per process, by tests/test_tdvp.py (the seeding has
to happen before the first ``import tenpy``).

    python tests/dropin/run_tdvp.py fake|cuda CASE

Prints one JSON line: {'reference_engine': record, 'fast_engine': record}.  tests/golden/make_golden_tdvp.py runs the same
cases with the plain reference.  Only gauge-independent quantities are recorded: <Sz> or <N> per site, the energy
``H_MPO.expectation_value``, the entanglement entropies, the bond dimensions, ``psi.norm`` and the Loschmidt amplitude
<psi(0)|psi(t)>.
"""
import json
import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings('ignore')

DT = 0.05
N_STEPS = 8
TRUNC = {'chi_max': 64, 'svd_min': 1.e-10}
CASES = ['xxz', 'tfi', 'hub', 'nnn', 'haldane', 'xxz_1site']


def model_case(name):
    """(model, product state, N_steps, observable) of a case, on the reference's model classes"""
    if name in ('xxz', 'xxz_1site'):
        from tenpy.models.spins import SpinChain
        return SpinChain(dict(L=10, S=0.5, Jx=1., Jy=1., Jz=1.3, hz=0., bc_MPS='finite', conserve='Sz')), \
            ['up', 'down'] * 5, N_STEPS, 'Sz'
    if name == 'tfi':
        from tenpy.models.tf_ising import TFIChain
        return TFIChain(dict(L=10, J=1., g=1.2, bc_MPS='finite', conserve=None)), ['up'] * 10, N_STEPS, 'Sz'
    if name == 'hub':
        from tenpy.models.hubbard import FermiHubbardChain
        return FermiHubbardChain(dict(L=6, t=1., U=3., mu=0., bc_MPS='finite', cons_N='N', cons_Sz='Sz')), \
            ['up', 'down'] * 3, N_STEPS, 'Ntot'
    if name == 'nnn':
        from tenpy.models.spins_nnn import SpinChainNNN2
        return SpinChainNNN2(dict(L=10, S=0.5, Jx=1., Jy=1., Jz=1., Jxp=0.5, Jyp=0.5, Jzp=0.5, hz=0.1,
                                  bc_MPS='finite', conserve='Sz')), ['up', 'down'] * 5, N_STEPS, 'Sz'
    if name == 'haldane':
        from tenpy.models.haldane import FermionicHaldaneModel
        M = FermionicHaldaneModel(dict(Lx=2, Ly=3, bc_MPS='finite', bc_y='cylinder', conserve='N', V=0.5))
        return M, ['full', 'empty'] * (M.lat.N_sites // 2), 4, 'N'
    raise ValueError(name)


def options():
    return {'dt': DT, 'N_steps': N_STEPS, 'trunc_params': dict(TRUNC)}


def run_case(name, TwoSite=None, SingleSite=None):
    """the case `name` with the TDVP engine classes `TwoSite` / `SingleSite` (default: the reference's)"""
    import numpy as np
    from tenpy.algorithms import tdvp
    from tenpy.networks.mps import MPS
    TwoSite = TwoSite or tdvp.TwoSiteTDVPEngine
    SingleSite = SingleSite or tdvp.SingleSiteTDVPEngine
    M, state, n_steps, op = model_case(name)
    psi0 = MPS.from_product_state(M.lat.mps_sites(), state, bc='finite')
    psi = psi0.copy()
    if name == 'xxz_1site':
        TwoSite(psi, M, dict(options(), N_steps=4)).run()
        eng = SingleSite(psi, M, dict(options(), N_steps=n_steps))
    else:
        eng = TwoSite(psi, M, dict(options(), N_steps=n_steps))
    eng.run()
    amp = complex(psi0.overlap(psi))
    return {'obs': [float(x) for x in np.real(psi.expectation_value(op))],
            'E': float(np.real(M.H_MPO.expectation_value(psi))),
            'S': [float(x) for x in psi.entanglement_entropy()],
            'chi': [int(c) for c in psi.chi],
            'norm': float(psi.norm),
            'amp': [amp.real, amp.imag],
            'time': float(np.real(eng.evolved_time))}


def main(mode, name):
    from run_reference_drivers import setup
    dropin = setup(mode)
    if mode == 'fake':
        sys.path.insert(0, os.path.dirname(HERE))
        import fake_krylov_combine
        import fake_mid_contract_z
        from tenpy_b200 import backend
        fake_krylov_combine.install(backend.get_lib())
        fake_mid_contract_z.install(backend.get_lib())
    out = {'reference_engine': run_case(name),
           'fast_engine': run_case(name, dropin.fast_tdvp_engine(), dropin.fast_tdvp_engine(single_site=True))}
    if mode == 'fake':
        from tenpy_b200 import backend
        out['krylov_combine_calls'] = backend.get_lib().calls.get('krylov_combine', 0)
    print(json.dumps(out))


if __name__ == '__main__':
    main(sys.argv[1], sys.argv[2])
