"""Matrix product operator and the environments of ``<psi|H|psi>``.

Minimal mirror of the reference ``tenpy/networks/mpo.py``: `MPO` (:72; tensors ``W[i]`` with labels
``'wL', 'wR', 'p', 'p*'``, `IdL` / `IdR` indices) and `MPOEnvironment` (:2740) with the four contraction
routines on the DMRG path -- `_contract_LP` (:3087), `_contract_RP` (:3097), `_contract_LHeff` (:3107),
`_contract_RHeff` (:3118) -- plus `full_contraction` (:3065).  All `L` environments stay resident in HBM
(the reference spills them to disk, tools/cache.py; 80 GB make that unnecessary here).
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import numpy as np

from ..linalg import np_conserved as npc
from ..linalg.charges import LegCharge

__all__ = ['MPO', 'MPOEnvironment']


class MPO:
    """Finite MPO with identical bond structure on every site (reference mpo.py:72)."""

    def __init__(self, sites, Ws, IdL, IdR, bc='finite'):
        self.sites = list(sites)
        self.L = len(self.sites)
        self.bc = bc
        self.finite = True
        self.dtype = np.float64
        self.chinfo = self.sites[0].leg.chinfo
        self._W = [W.itranspose(['wL', 'wR', 'p', 'p*']) for W in Ws]
        self.IdL = list(IdL) if isinstance(IdL, (list, tuple)) else [IdL] * (self.L + 1)
        self.IdR = list(IdR) if isinstance(IdR, (list, tuple)) else [IdR] * (self.L + 1)
        self.explicit_plus_hc = False

    @classmethod
    def from_grids(cls, sites, grids, w_charges, IdL, IdR):
        """Build from operator grids.

        grids[i][a][b] is ``None`` or a list of ``(coefficient, opname)``; `w_charges` is a list (length
        L+1) of (D, qnumber) charge tables of the MPO bonds (``None`` for no charges).  The MPO legs are
        *not bunched*: every MPO index is its own charge sector, like the reference's MPO legs."""
        sites = list(sites)
        chinfo = sites[0].leg.chinfo
        Ws = []
        for i, (site, grid) in enumerate(zip(sites, grids)):
            D1, D2 = len(grid), len(grid[0])
            dense = np.zeros((D1, D2, site.dim, site.dim))
            for a in range(D1):
                for b in range(D2):
                    if grid[a][b] is None:
                        continue
                    for coef, name in grid[a][b]:
                        dense[a, b] += coef * site.get_dense(name)
            if chinfo.qnumber == 0:
                legL = LegCharge.from_trivial(D1, chinfo, +1)
                legR = LegCharge.from_trivial(D2, chinfo, -1)
            else:
                legL = LegCharge.from_qind(chinfo, np.arange(D1 + 1), w_charges[i], +1)
                legR = LegCharge.from_qind(chinfo, np.arange(D2 + 1), w_charges[i + 1], -1)
            Ws.append(npc.Array.from_ndarray(dense, [legL, legR, site.leg, site.leg.conj()],
                                             labels=['wL', 'wR', 'p', 'p*'], qtotal=None, cutoff=1e-15))
        return cls(sites, Ws, IdL, IdR)

    @property
    def chi(self):
        return [W.get_leg('wL').ind_len for W in self._W] + [self._W[-1].get_leg('wR').ind_len]

    def get_W(self, i):
        return self._W[i]

    def get_IdL(self, i):
        return self.IdL[i]

    def get_IdR(self, i):
        return self.IdR[i + 1]


class MPOEnvironment:
    """Left / right parts ``LP[i]``, ``RP[i]`` of the network ``<bra|H|ket>`` (reference mpo.py:2740).

    ``LP[i]`` (labels ``'vR*', 'wR', 'vR'``) contains everything strictly left of site `i`,
    ``RP[i]`` (labels ``'vL', 'wL', 'vL*'``) everything strictly right of site `i`."""

    def __init__(self, bra, H, ket, **init_env_data):
        if ket is None:
            ket = bra
        self.bra, self.ket, self.H = bra, ket, H
        self.L = ket.L
        self.finite = True
        self.dtype = np.float64
        self._LP = [None] * self.L
        self._RP = [None] * self.L
        self._LP_age = [None] * self.L
        self._RP_age = [None] * self.L
        self.init_first_LP_last_RP(**init_env_data)

    def init_first_LP_last_RP(self, init_LP=None, init_RP=None, age_LP=0, age_RP=0):
        if init_LP is None:
            init_LP = self.init_LP(0)
        if init_RP is None:
            init_RP = self.init_RP(self.L - 1)
        self.set_LP(0, init_LP, age_LP)
        self.set_RP(self.L - 1, init_RP, age_RP)

    def init_LP(self, i):
        """trivial left part: identity on the virtual legs, unit vector `IdL` on the MPO leg (mpo.py:2893)"""
        leg_ket = self.ket.get_B(i, None).get_leg('vL')
        leg_mpo = self.H.get_W(i).get_leg('wL').conj()
        chi, D = leg_ket.ind_len, leg_mpo.ind_len
        dense = np.zeros((chi, D, chi))
        dense[:, self.H.get_IdL(i), :] = np.eye(chi)
        return npc.Array.from_ndarray(dense, [leg_ket, leg_mpo, leg_ket.conj()], labels=['vR*', 'wR', 'vR'],
                                      cutoff=0.5)

    def init_RP(self, i):
        leg_ket = self.ket.get_B(i, None).get_leg('vR')
        leg_mpo = self.H.get_W(i).get_leg('wR').conj()
        chi, D = leg_ket.ind_len, leg_mpo.ind_len
        dense = np.zeros((chi, D, chi))
        dense[:, self.H.get_IdR(i), :] = np.eye(chi)
        return npc.Array.from_ndarray(dense, [leg_ket, leg_mpo, leg_ket.conj()], labels=['vL*', 'wL', 'vL'],
                                      cutoff=0.5).itranspose(['vL', 'wL', 'vL*'])

    # ------------------------------------------------------------------ cache of parts
    def get_LP(self, i, store=True):
        """``LP[i]``, contracted from the nearest stored part on the left if necessary (mps.py:6429)."""
        i0 = i
        while self._LP[i0] is None:
            i0 -= 1
            if i0 < 0:
                raise ValueError('no left part found')
        LP, age = self._LP[i0], self._LP_age[i0]
        for j in range(i0, i):
            LP = self._contract_LP(j, LP)
            age += 1
            if store:
                self.set_LP(j + 1, LP, age)
        return LP

    def get_RP(self, i, store=True):
        i0 = i
        while self._RP[i0] is None:
            i0 += 1
            if i0 >= self.L:
                raise ValueError('no right part found')
        RP, age = self._RP[i0], self._RP_age[i0]
        for j in range(i0, i, -1):
            RP = self._contract_RP(j, RP)
            age += 1
            if store:
                self.set_RP(j - 1, RP, age)
        return RP

    def has_LP(self, i):
        return self._LP[i] is not None

    def has_RP(self, i):
        return self._RP[i] is not None

    def get_LP_age(self, i):
        return self._LP_age[i]

    def get_RP_age(self, i):
        return self._RP_age[i]

    def set_LP(self, i, LP, age):
        self._LP[i] = LP
        self._LP_age[i] = age

    def set_RP(self, i, RP, age):
        self._RP[i] = RP
        self._RP_age[i] = age

    def del_LP(self, i):
        self._LP[i] = None
        self._LP_age[i] = None

    def del_RP(self, i):
        self._RP[i] = None
        self._RP_age[i] = None

    def clear(self):
        """delete all parts except the boundary ones"""
        for i in range(1, self.L):
            self.del_LP(i)
        for i in range(self.L - 1):
            self.del_RP(i)

    # ------------------------------------------------------------------ contractions
    def _contract_LP(self, i, LP):
        """``LP[i] -> LP[i+1]`` (reference mpo.py:3087)"""
        LP = npc.tensordot(LP, self.ket.get_B(i, form='A'), axes=('vR', 'vL'))
        LP = npc.tensordot(self.H.get_W(i), LP, axes=(['p*', 'wL'], ['p', 'wR']))
        LP = npc.tensordot(self.bra.get_B(i, form='A').conj(), LP, axes=(['p*', 'vL*'], ['p', 'vR*']))
        return LP  # labels 'vR*', 'wR', 'vR'

    def _contract_RP(self, i, RP):
        """``RP[i] -> RP[i-1]`` (reference mpo.py:3097)"""
        RP = npc.tensordot(self.ket.get_B(i, form='B'), RP, axes=('vR', 'vL'))
        RP = npc.tensordot(RP, self.H.get_W(i), axes=(['p', 'wL'], ['p*', 'wR']))
        RP = npc.tensordot(RP, self.bra.get_B(i, form='B').conj(), axes=(['p', 'vL*'], ['p*', 'vR*']))
        return RP  # labels 'vL', 'wL', 'vL*'

    def _contract_LHeff(self, i, label_p='p0', pipe=None):
        """``LHeff = combine_legs(LP[i] . W[i])`` with legs ``'(vR*.p0)', 'wR', '(vR.p0*)'`` (mpo.py:3107)"""
        LP = self.get_LP(i)
        p, ps = label_p, label_p + '*'
        W = self.H.get_W(i).replace_labels(['p', 'p*'], [p, ps])
        LHeff = npc.tensordot(LP, W, axes=['wR', 'wL'])
        if pipe is None:
            pipe = LHeff.make_pipe(['vR*', p], qconj=+1)
        return LHeff.combine_legs([['vR*', p], ['vR', ps]], pipes=[pipe, pipe.conj()], new_axes=[0, 2])

    def _contract_RHeff(self, i, label_p='p1', pipe=None):
        """``RHeff`` with legs ``'wL', '(p1*.vL)', '(p1.vL*)'`` (mpo.py:3118)"""
        RP = self.get_RP(i)
        p, ps = label_p, label_p + '*'
        W = self.H.get_W(i).replace_labels(['p', 'p*'], [p, ps])
        RHeff = npc.tensordot(W, RP, axes=['wR', 'wL'])
        if pipe is None:
            pipe = RHeff.make_pipe([p, 'vL*'], qconj=-1)
        return RHeff.combine_legs([[p, 'vL*'], [ps, 'vL']], pipes=[pipe, pipe.conj()], new_axes=[2, 1])

    def full_contraction(self, i0):
        """``<bra|H|ket>`` contracted at the bond right of site `i0` (reference mpo.py:3064 on top of
        `MPSEnvironment._full_contraction_LP_RP`, mps.py:6706): ``LP[i0+1]`` and ``RP[i0]`` with the bond matrix
        (1-D Schmidt values, or the 2-D matrix a mixer leaves) of bra and ket in between."""
        if i0 + 1 == self.L:
            LP = self._contract_LP(i0, self.get_LP(i0, store=False))
        else:
            LP = self.get_LP(i0 + 1, store=False)
        S_bra = self.bra.get_SR(i0)
        if isinstance(S_bra, npc.Array):
            LP = npc.tensordot(S_bra.conj(), LP, axes=['vL*', 'vR*'])
        else:
            LP = LP.scale_axis(S_bra, 'vR*')
        S_ket = self.ket.get_SR(i0)
        if isinstance(S_ket, npc.Array):
            LP = npc.tensordot(LP, S_ket, axes=['vR', 'vL'])
        else:
            LP = LP.scale_axis(S_ket, 'vR')
        RP = self.get_RP(i0, store=False)
        res = npc.inner(LP, RP, axes=[['vR*', 'wR', 'vR'], ['vL*', 'wL', 'vL']], do_conj=False)
        if self.H.explicit_plus_hc:
            res = res + np.conj(res)
        return res
