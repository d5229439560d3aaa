"""The three benchmark chains as explicit MPOs (cold path, host side).

The reference builds these through its generic `CouplingMPOModel` machinery (``tenpy/models/model.py``,
``tf_ising.py:74`` `TFIChain`, ``spins.py`` `SpinChain`, ``hubbard.py:207`` `FermiHubbardChain`); model
construction is outside the hot path (SURVEY.md section 2, rows 16-17), so here each Hamiltonian is written
down directly as its finite-state-machine MPO.  The resulting bond dimensions equal the reference's
(TFI D=3, XXZ D=5, Hubbard D=6) and energies are pinned against the reference in tests/golden.

* TFIChain:          ``H = -J sum_i sx_i sx_{i+1} - g sum_i sz_i``  (Pauli matrices)
* SpinChain (S=1/2): ``H = sum_i Jx Sx Sx + Jy Sy Sy + Jz Sz Sz + D (Sx Sy - Sy Sx) - hz sum_i Sz_i``
* FermiHubbardChain: ``H = -t sum_{i,s} (c^+_{i,s} c_{i+1,s} + h.c.) + U sum_i n_up n_dn - mu sum_i n_i``
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import numpy as np

from .networks.site import SpinHalfSite, SpinHalfFermionSite
from .networks.mpo import MPO

__all__ = ['TFIChain', 'SpinChain', 'XXZChain', 'FermiHubbardChain']


class _ChainModel:
    """holds `lat_sites` and `H_MPO` (the attributes the DMRG engine reads from a reference model)"""

    def __init__(self, sites, grid, op_names_first_row, IdL, IdR):
        self.sites = sites
        self.L = len(sites)
        site = sites[0]
        chinfo = site.leg.chinfo
        D = len(grid)
        if chinfo.qnumber:
            # charge of MPO index b = charge of the operator in W[0, b] (IdL row); see mpo.MPO.from_grids
            wq = np.zeros((D, chinfo.qnumber), dtype=np.int64)
            for b, name in enumerate(op_names_first_row):
                if name is not None:
                    wq[b] = site.op_charge(name)
            w_charges = [chinfo.make_valid(wq)] * (self.L + 1)
        else:
            w_charges = [None] * (self.L + 1)
        self.H_MPO = MPO.from_grids(sites, [grid] * self.L, w_charges, IdL, IdR)
        self.lat_sites = sites
        self._grid, self._IdL, self._IdR = grid, IdL, IdR
        self._H_bond = None

    @property
    def H_bond(self):
        """Nearest-neighbour bond terms, ``H_bond[j]`` acting on sites ``(j-1, j)``, ``H_bond[0] = None``.

        Same decomposition as the reference's `calc_H_bond_from_MPO` (``tenpy/models/model.py:752``): the
        two-site part is ``sum_b W[IdL, b] (x) W[b, IdR]``; the onsite term ``W[IdL, IdR]`` of a site is shared
        half-half between its two bonds, fully at the chain ends.  Arrays with labels ``p0, p0*, p1, p1*``."""
        if self._H_bond is None:
            from .linalg import np_conserved as npc
            grid, IdL, IdR, L = self._grid, self._IdL, self._IdR, self.L
            site = self.sites[0]
            d = site.dim

            def dense(entry):
                res = np.zeros((d, d))
                for coef, name in (entry or []):
                    res = res + coef * site.get_dense(name)
                return res

            onsite = dense(grid[IdL][IdR])
            pair = np.zeros((d, d, d, d))
            for b in range(len(grid)):
                if b in (IdL, IdR):
                    continue
                pair += np.einsum('ij,kl->ijkl', dense(grid[IdL][b]), dense(grid[b][IdR]))
            one = np.eye(d)
            legs = [site.leg, site.leg.conj(), site.leg, site.leg.conj()]
            H_bond = [None] * L
            for j in range(1, L):
                s_i = 1. if j - 1 == 0 else 0.5
                s_j = 1. if j == L - 1 else 0.5
                h = pair + s_i * np.einsum('ij,kl->ijkl', onsite, one) + s_j * np.einsum('ij,kl->ijkl', one, onsite)
                H_bond[j] = npc.Array.from_ndarray(h, legs, labels=['p0', 'p0*', 'p1', 'p1*'], cutoff=1e-16)
            self._H_bond = H_bond
        return self._H_bond

    def bond_energies(self, psi):
        """``<psi| H_bond[j] |psi>`` for ``j = 1 .. L-1`` (reference model.py `NearestNeighborModel.bond_energies`
        :706); needs `psi` in canonical form around each bond."""
        from .linalg import np_conserved as npc
        E = []
        for j in range(1, self.L):
            theta = psi.get_theta(j - 1, n=2)
            Hth = npc.tensordot(self.H_bond[j], theta, axes=(['p0*', 'p1*'], ['p0', 'p1']))
            E.append(float(npc.inner(theta, Hth, axes='labels', do_conj=True)))
        return np.array(E)


class TFIChain(_ChainModel):
    """Transverse field Ising chain (reference tf_ising.py:74); params ``L, J, g, conserve``."""

    def __init__(self, params):
        L = params['L']
        J, g = params.get('J', 1.), params.get('g', 1.)
        conserve = params.get('conserve', None)
        if params.get('bc_MPS', 'finite') != 'finite':
            raise NotImplementedError('finite chains only')
        site = SpinHalfSite(conserve=conserve)
        grid = [[[(1., 'Id')], [(1., 'Sigmax')], [(-g, 'Sigmaz')]],
                [None, None, [(-J, 'Sigmax')]],
                [None, None, [(1., 'Id')]]]
        _ChainModel.__init__(self, [site] * L, grid, ['Id', 'Sigmax', None], 0, 2)


class SpinChain(_ChainModel):
    """Spin-1/2 chain (reference spins.py `SpinChain`, S=0.5); params ``L, Jx, Jy, Jz, hz, D, conserve``.

    `D`: z-axis Dzyaloshinskii-Moriya coupling ``D sum_i (Sx_i Sy_{i+1} - Sy_i Sx_{i+1})
    = (iD/2) sum_i (S+_i S-_{i+1} - S-_i S+_{i+1})``; it conserves Sz when ``Jx == Jy``.  A non-zero `D` makes the MPO
    complex (ComplexArray tensors); with ``D = 0`` it is the real MPO."""

    def __init__(self, params):
        L = params['L']
        if params.get('S', 0.5) != 0.5:
            raise NotImplementedError('S=1/2 only')
        Jx, Jy, Jz = params.get('Jx', 1.), params.get('Jy', 1.), params.get('Jz', 1.)
        hz = params.get('hz', 0.)
        D = params.get('D', 0.)
        conserve = params.get('conserve', 'best')
        if conserve == 'best':
            conserve = 'Sz' if Jx == Jy else 'parity'
        if conserve == 'Sz' and Jx != Jy:
            raise ValueError('Sz is not conserved for Jx != Jy')
        site = SpinHalfSite(conserve=conserve)
        jpm = (Jx + Jy) / 4.
        jpp = (Jx - Jy) / 4.
        dm = 0.5j * D          # S+_i S-_{i+1} gets +iD/2, S-_i S+_{i+1} gets -iD/2
        last = [[(-hz, 'Sz')] if hz != 0. else None,
                [(jpm + dm if D != 0. else jpm, 'Sm')] + ([(jpp, 'Sp')] if jpp != 0. else []),
                [(jpm - dm if D != 0. else jpm, 'Sp')] + ([(jpp, 'Sm')] if jpp != 0. else []),
                [(Jz, 'Sz')],
                [(1., 'Id')]]
        grid = [[[(1., 'Id')], [(1., 'Sp')], [(1., 'Sm')], [(1., 'Sz')], last[0]],
                [None, None, None, None, last[1]],
                [None, None, None, None, last[2]],
                [None, None, None, None, last[3]],
                [None, None, None, None, last[4]]]
        _ChainModel.__init__(self, [site] * L, grid, ['Id', 'Sp', 'Sm', 'Sz', None], 0, 4)


class XXZChain(SpinChain):
    """``H = Jxx/2 (S+S- + h.c.) + Jz Sz Sz - hz Sz`` (reference xxz_chain.py)."""

    def __init__(self, params):
        p = dict(params)
        Jxx = p.pop('Jxx', 1.)
        p.setdefault('Jz', 1.)
        p['Jx'] = p['Jy'] = Jxx
        p.setdefault('conserve', 'Sz')
        SpinChain.__init__(self, p)


class FermiHubbardChain(_ChainModel):
    """Spinful Fermi-Hubbard chain (reference hubbard.py:207); params ``L, t, U, mu, cons_N, cons_Sz``.

    Jordan-Wigner: ``c^+_i c_{i+1} = (Cd JW)_i (C)_{i+1}``, ``c^+_{i+1} c_i = (JW C)_i (Cd)_{i+1}``."""

    def __init__(self, params):
        L = params['L']
        t, U, mu = params.get('t', 1.), params.get('U', 0.), params.get('mu', 0.)
        site = SpinHalfFermionSite(cons_N=params.get('cons_N', 'N'), cons_Sz=params.get('cons_Sz', 'Sz'))
        d = site.get_dense
        site.add_op('CduJW', d('Cdu') @ d('JW'), permute=False)
        site.add_op('JWCu', d('JW') @ d('Cu'), permute=False)
        site.add_op('CddJW', d('Cdd') @ d('JW'), permute=False)
        site.add_op('JWCd', d('JW') @ d('Cd'), permute=False)
        onsite = [(U, 'NuNd')] + ([(-mu, 'Ntot')] if mu != 0. else [])
        if U == 0. and mu == 0.:
            onsite = None
        grid = [[[(1., 'Id')], [(1., 'CduJW')], [(1., 'JWCu')], [(1., 'CddJW')], [(1., 'JWCd')], onsite],
                [None, None, None, None, None, [(-t, 'Cu')]],
                [None, None, None, None, None, [(-t, 'Cdu')]],
                [None, None, None, None, None, [(-t, 'Cd')]],
                [None, None, None, None, None, [(-t, 'Cdd')]],
                [None, None, None, None, None, [(1., 'Id')]]]
        _ChainModel.__init__(self, [site] * L, grid, ['Id', 'CduJW', 'JWCu', 'CddJW', 'JWCd', None], 0, 5)
