#!/usr/bin/env python
"""The complex drop-in case of run_dmrg_complex.py (the reference's ``FermionicHaldaneModel`` through
``dropin.fast_two_site_engine()``) with the split-order matvec forced on every bond.  Executed in its own process by
tests/test_complex_split_matvec.py.

    python tests/dropin/run_dmrg_complex_split.py fake|cuda

Prints one JSON line: {'fast_engine': {'E', 'S', 'chi', ...}, 'identity_env_bonds': n}.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from run_dmrg_complex import run_case  # noqa: E402


def main(mode):
    from run_reference_drivers import setup
    dropin = setup(mode)
    if mode == 'fake':
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        from fake_mid_contract_z import install
        from tenpy_b200 import backend
        install(backend.get_lib())
    from tenpy_b200.algorithms.mps_common import SplitOrderMatvec
    SplitOrderMatvec.matvec_order = 'split'
    n0 = SplitOrderMatvec.stats['identity_env_bonds']
    out = {'fast_engine': run_case(dropin.fast_two_site_engine())}
    out['identity_env_bonds'] = SplitOrderMatvec.stats['identity_env_bonds'] - n0
    print(json.dumps(out))


if __name__ == '__main__':
    main(sys.argv[1])
