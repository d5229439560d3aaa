"""Local Hilbert spaces of the benchmark chains (host-side, cold path).

Minimal mirror of the reference ``tenpy/networks/site.py`` (`Site`, `SpinHalfSite`,
`SpinHalfFermionSite`): a site is a physical `leg` (LegCharge) plus named on-site operators given as
dense ``(d, d)`` matrices in the (possibly charge-sorted) basis of the leg; operators are converted to
device Arrays with labels ``'p', 'p*'`` on demand.  Charge values follow the reference's conventions
(``2*Sz`` for spins, ``N`` and ``2*Sz`` for fermions, Z2 parity where requested).
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import numpy as np

from ..linalg import np_conserved as npc
from ..linalg.charges import ChargeInfo, LegCharge

__all__ = ['Site', 'SpinHalfSite', 'SpinHalfFermionSite']


class Site:
    """Physical leg + on-site operators (reference site.py `Site`).

    `ops` maps name -> dense (d, d) ndarray given in the *original* state order `state_labels`; if
    `sort_charge`, the basis is permuted such that the leg is sorted by charge (as the reference does)."""

    def __init__(self, leg, state_labels, sort_charge=True, **ops):
        self.dim = leg.ind_len
        self.perm = np.arange(self.dim)
        if sort_charge and leg.chinfo.qnumber > 0:
            qflat = leg.to_qflat()
            self.perm = np.lexsort(qflat.T)
            leg = LegCharge.from_qflat(leg.chinfo, qflat[self.perm], leg.qconj)
        self.leg = leg
        inv = np.argsort(self.perm)
        self.state_labels = {str(lab): int(inv[i]) for i, lab in enumerate(state_labels)}
        self.opnames = set()
        self._dense = {}
        self._npc = {}
        for name, op in ops.items():
            self.add_op(name, op)
        if 'Id' not in self._dense:
            self.add_op('Id', np.eye(self.dim), permute=False)

    def add_op(self, name, op, permute=True):
        """`op`: dense (d, d); real (float64) unless it has a non-zero imaginary part (complex128)"""
        op = np.asarray(op)
        op = op.astype(np.complex128 if np.iscomplexobj(op) and np.any(op.imag != 0.) else np.float64)
        if permute:
            op = op[np.ix_(self.perm, self.perm)]
        self._dense[name] = op
        self.opnames.add(name)

    def get_dense(self, name):
        return self._dense[name]

    def op_charge(self, name):
        """charge ``q_p - q_p*`` carried by operator `name` (must be unique)."""
        op = self._dense[name]
        qflat = self.leg.to_qflat() * self.leg.qconj
        r, c = np.nonzero(np.abs(op) > 1e-14)
        if len(r) == 0:
            return self.leg.chinfo.make_valid()
        dq = self.leg.chinfo.make_valid(qflat[r] - qflat[c])
        if np.any(dq != dq[0]):
            raise ValueError('operator {0} does not have a well-defined charge'.format(name))
        return dq[0]

    def get_op(self, name):
        """device Array (a ComplexArray for a complex operator) with labels ``'p', 'p*'``"""
        if name not in self._npc:
            cls = npc.ComplexArray if np.iscomplexobj(self._dense[name]) else npc.Array
            self._npc[name] = cls.from_ndarray(self._dense[name], [self.leg, self.leg.conj()], labels=['p', 'p*'])
        return self._npc[name]

    def state_index(self, label):
        if isinstance(label, str):
            return self.state_labels[label]
        return int(np.argsort(self.perm)[int(label)])


class SpinHalfSite(Site):
    """Spin-1/2 site; states ``'up', 'down'``; ``conserve`` in {'Sz', 'parity', None} (reference site.py)."""

    def __init__(self, conserve='Sz', sort_charge=True):
        Sx = np.array([[0., 0.5], [0.5, 0.]])
        Sz = np.array([[0.5, 0.], [0., -0.5]])
        Sp = np.array([[0., 1.], [0., 0.]])
        Sm = np.array([[0., 0.], [1., 0.]])
        ops = dict(Sp=Sp, Sm=Sm, Sz=Sz, Sigmaz=2. * Sz)
        if conserve == 'Sz':
            chinfo = ChargeInfo([1], ['2*Sz'])
            leg = LegCharge.from_qflat(chinfo, [1, -1])
        else:
            ops.update(Sx=Sx, Sigmax=2. * Sx)
            if conserve == 'parity':
                chinfo = ChargeInfo([2], ['parity_Sz'])
                leg = LegCharge.from_qflat(chinfo, [1, 0])
            else:
                leg = LegCharge.from_trivial(2)
        self.conserve = conserve
        Site.__init__(self, leg, ['up', 'down'], sort_charge=sort_charge, **ops)


class SpinHalfFermionSite(Site):
    """Spinful fermions; states ``'empty', 'up', 'down', 'full'`` (reference site.py `SpinHalfFermionSite`).

    Operators (Jordan-Wigner strings are handled by the MPO builder): ``Cu, Cdu, Cd, Cdd, Nu, Nd, Ntot,
    NuNd, JW, JWu, JWd``.  ``Cd`` already contains the on-site sign ``JWu`` like the reference."""

    def __init__(self, cons_N='N', cons_Sz='Sz', sort_charge=True):
        d = 4
        Nu_diag = np.array([0., 1., 0., 1.])
        Nd_diag = np.array([0., 0., 1., 1.])
        Nu, Nd = np.diag(Nu_diag), np.diag(Nd_diag)
        JWu = np.diag(1. - 2 * Nu_diag)
        JWd = np.diag(1. - 2 * Nd_diag)
        JW = JWu @ JWd
        Cu = np.zeros((d, d))
        Cu[0, 1] = Cu[2, 3] = 1.
        Cd_noJW = np.zeros((d, d))
        Cd_noJW[0, 2] = Cd_noJW[1, 3] = 1.
        Cd = JWu @ Cd_noJW
        ops = dict(JW=JW, JWu=JWu, JWd=JWd, Cu=Cu, Cdu=Cu.T.copy(), Cd=Cd, Cdd=Cd.T.copy(), Nu=Nu, Nd=Nd,
                   Ntot=Nu + Nd, NuNd=Nu @ Nd, Sz=0.5 * (Nu - Nd))
        qmod, qnames, charges = [], [], []
        if cons_N == 'N':
            qmod.append(1), qnames.append('N'), charges.append([0, 1, 1, 2])
        elif cons_N == 'parity':
            qmod.append(2), qnames.append('parity_N'), charges.append([0, 1, 1, 0])
        if cons_Sz == 'Sz':
            qmod.append(1), qnames.append('2*Sz'), charges.append([0, 1, -1, 0])
        elif cons_Sz == 'parity':
            qmod.append(4), qnames.append('parity_Sz'), charges.append([0, 1, 3, 0])
        if len(qmod) == 0:
            leg = LegCharge.from_trivial(d)
        else:
            leg = LegCharge.from_qflat(ChargeInfo(qmod, qnames), np.array(charges).T)
        self.cons_N, self.cons_Sz = cons_N, cons_Sz
        Site.__init__(self, leg, ['empty', 'up', 'down', 'full'], sort_charge=sort_charge, **ops)
