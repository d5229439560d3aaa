#!/usr/bin/env python
"""Golden numbers of ground-state DMRG of a complex Hamiltonian, generated with the UNMODIFIED reference on its own NumPy
engine (build container only):

    TENPY_NO_CYTHON=1 PYTHONPATH=/root/reference python tests/golden/make_golden_dmrg_complex.py

Runs the case of tests/dropin/run_dmrg_complex.py (``FermionicHaldaneModel``, Lx = 2, Ly = 3, cylinder, N conserved,
V = 0.5, two-site DMRG with the mixer, chi_max = 64) and stores E, all entanglement entropies and the bond dimensions in
dmrg_complex.npz, together with the exact ground-state energy of the half-filled sector (N = 6, dimension 924) from the
reference's dense ``ExactDiag`` of the same MPO."""
import os
import sys
import warnings

import numpy as np

os.environ.setdefault('TENPY_NO_CYTHON', '1')
sys.path.insert(0, os.environ.get('TENPY_REFERENCE', '/root/reference'))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'dropin'))
warnings.simplefilter('ignore')
import tenpy.linalg.np_conserved as npc  # noqa: E402
assert not npc.__name__.startswith('tenpy_b200'), 'must run with the plain reference'
from tenpy.algorithms.exact_diag import ExactDiag  # noqa: E402
from tenpy.models.haldane import FermionicHaldaneModel  # noqa: E402
from run_dmrg_complex import MODEL, run_case  # noqa: E402

rec = run_case()
M = FermionicHaldaneModel(dict(MODEL))
ED = ExactDiag.from_H_mpo(M.H_MPO, charge_sector=[M.lat.N_sites // 2], max_size=1e8)
ED.build_full_H_from_mpo()
ED.full_diagonalization()
E_exact = float(np.min(ED.E))
dim = int(np.sum(ED._mask))
print('E', rec['E'], 'E_exact', E_exact, 'sector dimension', dim, 'chi', rec['chi'], 'S', rec['S'])
assert dim == 924
np.savez_compressed(os.path.join(HERE, 'dmrg_complex.npz'), E=rec['E'], S=np.array(rec['S']), chi=np.array(rec['chi']),
                    E_exact=E_exact, sector_dim=dim)
