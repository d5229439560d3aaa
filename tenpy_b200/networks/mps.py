"""Finite matrix product state in (mixed) canonical form: the part of the reference's MPS the DMRG path uses.

Minimal mirror of ``tenpy/networks/mps.py`` (`MPS` :1537): tensors ``B[i]`` with labels ``'vL', 'p', 'vR'``,
Schmidt values ``S[i]`` on the bond *left* of site ``i`` (``S[L]`` right of the last site), canonical `form`
per site (``'A' = (1, 0)``, ``'B' = (0, 1)``), `get_B` (:2882), `set_B` (:2939), `get_theta` (:3041),
`entanglement_entropy` (:3777).  During DMRG with a mixer a bond may temporarily hold a 2-D Array instead of
1-D Schmidt values (reference `_scale_axis_B`, mps.py:5964); only non-negative powers of it are ever needed
on the two-site path.  `S` vectors live on the host (they are tiny), tensors on the device.
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import numpy as np

from ..linalg import np_conserved as npc
from ..linalg.charges import LegCharge

__all__ = ['MPS']


class MPS:
    _valid_forms = {'A': (1., 0.), 'C': (0.5, 0.5), 'B': (0., 1.), 'G': (0., 0.), 'Th': (1., 1.), None: None}
    _B_labels = ['vL', 'p', 'vR']

    def __init__(self, sites, Bs, SVs, bc='finite', form='B', norm=1.):
        if bc != 'finite':
            raise NotImplementedError('only finite MPS')
        self.sites = list(sites)
        self.L = len(self.sites)
        self.bc = bc
        self.finite = True
        self.chinfo = self.sites[0].leg.chinfo
        self.norm = norm
        self.form = [self._to_valid_form(form)] * self.L if not isinstance(form, list) else \
            [self._to_valid_form(f) for f in form]
        self._B = [B.itranspose(self._B_labels) for B in Bs]
        self._S = [None if s is None else np.array(s, dtype=np.float64) for s in SVs]
        if len(self._S) != self.L + 1:
            raise ValueError('need L+1 singular value arrays')

    @property
    def dtype(self):
        """complex128 once a tensor is a ComplexArray (a product state is real; the first complex update makes it
        complex), else float64"""
        return np.complex128 if any(isinstance(B, npc.ComplexArray) for B in self._B) else np.float64

    def _to_valid_form(self, form):
        if isinstance(form, tuple):
            return form
        return self._valid_forms[form]

    @classmethod
    def from_product_state(cls, sites, p_state, bc='finite', dtype=np.float64, form='B', chargeL=None):
        """Product state; `p_state[i]` is a state label or index of site ``i`` (reference mps.py:1830)."""
        sites = list(sites)
        L = len(sites)
        chinfo = sites[0].leg.chinfo
        charge = chinfo.make_valid(chargeL)
        Bs, SVs = [], [np.ones(1)]
        for i, site in enumerate(sites):
            idx = site.state_index(p_state[i])
            legL = LegCharge.from_qflat(chinfo, [charge], qconj=+1)
            qi, _ = site.leg.get_qindex(idx)
            charge = chinfo.make_valid(charge + site.leg.get_charge(qi))
            legR = LegCharge.from_qflat(chinfo, [charge], qconj=-1)
            dense = np.zeros((1, site.dim, 1))
            dense[0, idx, 0] = 1.
            Bs.append(npc.Array.from_ndarray(dense, [legL, site.leg, legR], labels=['vL', 'p', 'vR']))
            SVs.append(np.ones(1))
        return cls(sites, Bs, SVs, bc, form)

    # ------------------------------------------------------------------
    @property
    def chi(self):
        """bond dimensions of the L-1 inner bonds"""
        return [self._B[i].get_leg('vR').ind_len for i in range(self.L - 1)]

    def get_SL(self, i):
        return self._S[i]

    def get_SR(self, i):
        return self._S[i + 1]

    def set_SL(self, i, S):
        self._S[i] = S

    def set_SR(self, i, S):
        self._S[i + 1] = S

    def set_B(self, i, B, form='B'):
        """Reference mps.py:2939; `form` as for `get_B`, e.g. ``'Th'`` for the one-site wave function the TDVP leaves on
        a site between two updates."""
        self.form[i] = self._to_valid_form(form)
        self._B[i] = B.itranspose(self._B_labels)

    def _scale_axis_B(self, B, S, form_diff, axis_B, cutoff=1e-16):
        """Reference mps.py:5964; `cutoff`: of the pseudo-inverse of a 2-D `S`."""
        if form_diff == 0.:
            return B
        if not isinstance(S, npc.Array):
            if form_diff == -1.:
                S = 1. / S
            elif form_diff != 1.:
                S = S**form_diff
            return B.scale_axis(S, axis_B)
        if form_diff == -1.:
            S = npc.pinv(S, cutoff)
        elif form_diff != 1.:
            raise ValueError("Can't scale/tensordot a 2D `S` for non-integer `form_diff`")
        if axis_B == 'vL':
            return npc.tensordot(S, B, axes=[1, 'vL']).ireplace_label(0, 'vL') if S._labels[0] != 'vL' else \
                npc.tensordot(S, B, axes=[1, 'vL'])
        B2 = npc.tensordot(B, S, axes=['vR', 0])
        if B2._labels[-1] != 'vR':
            B2.ireplace_label(B2.rank - 1, 'vR')
        return B2

    def get_B(self, i, form='B', copy=False, cutoff=1e-16, label_p=None):
        """Tensor of site `i` in the requested canonical form (reference mps.py:2882)."""
        new_form = self._to_valid_form(form)
        old_form = self.form[i]
        B = self._B[i]
        if copy:
            B = B.copy()
        if new_form is not None and old_form != new_form:
            if old_form is None:
                raise ValueError('can not convert a tensor without canonical form')
            fL, fR = new_form
            if fL is not None and fL != old_form[0]:
                B = self._scale_axis_B(B, self.get_SL(i), fL - old_form[0], 'vL', cutoff)
            if fR is not None and fR != old_form[1]:
                B = self._scale_axis_B(B, self.get_SR(i), fR - old_form[1], 'vR', cutoff)
        if label_p is not None:
            B = B.replace_label('p', 'p' + label_p)
        return B

    def get_theta(self, i, n=2, cutoff=1e-16, formL=1., formR=1.):
        """n-site wave function with labels ``vL, p0, ..., p{n-1}, vR`` (reference mps.py:3041); `cutoff`: of the
        pseudo-inverse of a 2-D bond matrix."""
        if n == 1:
            return self.get_B(i, (1., 1.), True, cutoff, '0')
        theta = self.get_B(i, (formL, None), False, cutoff, '0')
        old_fR = self.form[i][1]
        for k in range(1, n):
            new_fR = None if k + 1 < n else formR
            B = self.get_B(i + k, (1. - old_fR, new_fR), False, cutoff, str(k))
            old_fR = self.form[i + k][1]
            theta = npc.tensordot(theta, B, axes=['vR', 'vL'])
        return theta

    def entanglement_entropy(self, n=1, bonds=None):
        """von-Neumann (n=1) or Renyi entropies at the inner bonds (reference mps.py:3777)."""
        if bonds is None:
            bonds = range(1, self.L)
        res = []
        for ib in bonds:
            s = self._S[ib]
            if isinstance(s, npc.Array):
                s = np.linalg.svd(s.to_ndarray(), compute_uv=False)
            s = np.asarray(s)
            s = s[s > 1e-30]
            if n == 1:
                res.append(float(-np.sum(s**2 * np.log(s**2))))
            else:
                res.append(float(np.log(np.sum(s**(2 * n))) / (1. - n)))
        return np.array(res)

    def isometry_test(self):
        """max deviation of every site tensor from the isometry condition of its canonical form."""
        out = []
        for i in range(self.L):
            f = self.form[i]
            B = self._B[i]
            if f == (1., 0.):
                M = npc.tensordot(B.conj(), B, axes=[['vL*', 'p*'], ['vL', 'p']])
            elif f == (0., 1.):
                M = npc.tensordot(B, B.conj(), axes=[['p', 'vR'], ['p*', 'vR*']])
            else:
                out.append(np.nan)
                continue
            d = M.to_ndarray()
            out.append(float(np.max(np.abs(d - np.eye(d.shape[0])))))
        return np.array(out)

    def norm_test(self):
        """Canonical-form check of the reference (mps.py:4444): for each site the norm differences between the
        reduced density matrices of ``theta[i]`` and ``S[i]^2`` (left, column 0) / ``S[i+1]^2`` (right, column 1)."""
        err = np.empty((self.L, 2), dtype=float)
        for i in range(self.L):
            th = self.get_theta(i, 1)
            rho_L = npc.tensordot(th, th.conj(), axes=(['p0', 'vR'], ['p0*', 'vR*']))
            S = self.get_SL(i)
            if isinstance(S, npc.Array):
                rho_L2 = npc.tensordot(S, S.conj(), axes=['vR', 'vR*'])
            else:
                rho_L2 = npc.diag(S**2, rho_L.get_leg('vL'), labels=['vL', 'vL*'])
            err[i, 0] = npc.norm(rho_L - rho_L2)
            rho_R = npc.tensordot(th, th.conj(), axes=(['vL', 'p0'], ['vL*', 'p0*']))
            S = self.get_SR(i)
            if isinstance(S, npc.Array):
                rho_R2 = npc.tensordot(S, S.conj(), axes=['vL', 'vL*'])
            else:
                rho_R2 = npc.diag(S**2, rho_R.get_leg('vR'), labels=['vR', 'vR*'])
            err[i, 1] = npc.norm(rho_R - rho_R2)
        return err

    def canonical_form(self, renormalize=True, cutoff=0.):
        """Bring the finite MPS into right-canonical ``'B'`` form, in place (reference mps.py:4501
        `canonical_form_finite`): one sweep to the right orthonormalising, one sweep to the left computing all
        Schmidt values by SVDs.  The reference uses QR in the first sweep; here both sweeps use the batched
        block-Jacobi SVD (``Q = U``, ``R = S V``), which gives the same canonical form."""
        L = self.L
        assert L > 1
        self.set_SL(0, np.array([1.]))
        self.set_SR(L - 1, np.array([1.]))
        if any(f is None for f in self.form):
            M = self.get_B(0, form=None)
            form = None
        else:
            M = self.get_B(0, form='Th')
            form = 'B'
        M = self._normalize_array(M.copy(deep=True), renormalize)
        R = None
        for i in range(L - 1):
            if i > 0:
                M = npc.tensordot(R, self.get_B(i, form), axes=['vR', 'vL'])
                M = self._normalize_array(M, renormalize)
            Mc = M.combine_legs(['vL', 'p'])
            Q, s, V = npc.svd(Mc, cutoff=0., qtotal_LR=[None, Mc.qtotal], inner_labels=['vR', 'vL'])
            R = V.iscale_axis(s, 'vL')
            self.set_B(i, Q.split_legs(0), form='A')
        M = npc.tensordot(R, self.get_B(L - 1, form), axes=['vR', 'vL'])
        M = self._normalize_array(M, renormalize)
        U, S, V = npc.svd(M.combine_legs(['p', 'vR'], qconj=-1), cutoff=cutoff, inner_labels=['vR', 'vL'])
        if not renormalize:
            self.norm = self.norm * np.linalg.norm(S)
        S = S / np.linalg.norm(S)
        self.set_SL(L - 1, S)
        self.set_B(L - 1, V.split_legs(1), form='B')
        for i in range(L - 2, -1, -1):
            M = self.get_B(i, 'A')
            M = npc.tensordot(M, U.scale_axis(S, 'vR'), axes=['vR', 'vL'])
            U, S, V = npc.svd(M.combine_legs(['p', 'vR'], qconj=-1), cutoff=cutoff, qtotal_LR=[None, M.qtotal],
                              inner_labels=['vR', 'vL'])
            S = S / np.linalg.norm(S)
            self.set_SL(i, S)
            self.set_B(i, V.split_legs(1), form='B')
        assert len(S) == 1
        u = U.to_ndarray()[0, 0]                               # a sign (a phase for a complex state), kept like the
        self._B[0] *= u if isinstance(U, npc.ComplexArray) else float(u)      # reference does

    def _normalize_array(self, arr, renormalize):
        """Reference mps.py:6151."""
        nrm = npc.norm(arr)
        if not renormalize:
            self.norm = self.norm * nrm
        arr /= nrm
        return arr
