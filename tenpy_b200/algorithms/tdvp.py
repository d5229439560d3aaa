"""Real-time TDVP (time-dependent variational principle) of finite MPS on the H100-native tensor engine.

Host-side mirror of the reference driver ``tenpy/algorithms/tdvp.py`` (`TDVPEngine` :58, `TwoSiteTDVPEngine` :233,
`SingleSiteTDVPEngine` :318; the projector-splitting integrator of Haegeman et al., PRB 94, 165116 (2016)).  Same options
(``dt``, ``N_steps``, ``start_time``, ``preserve_norm``, ``trunc_params``, ``lanczos_params``, ``max_dt``, ``combine``),
same sweep schedules and update rules.  The sweep, the effective Hamiltonians and the environment updates are those of
the DMRG engine (:class:`~tenpy_b200.algorithms.dmrg.TwoSiteDMRGEngine`, which these engines subclass): the two-site step
uses the engine's `TwoSiteH`, so the ``'auto'`` matvec order chooses its route as in DMRG.  Each local step is
``expm(-i dt/2 H_eff) theta`` by :class:`~tenpy_b200.linalg.krylov_based.LanczosEvolution`: device-scalar Lanczos and
one ``b200_krylov_combine_f64`` for the result.

Not provided: Krylov subspace expansion (``Krylov_params['expansion_dim'] > 0``), infinite MPS, time-dependent
Hamiltonians and non-hermitian evolution (``lanczos_params['hermitian'] = False``, the reference's ArnoldiEvolution).
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import logging

import numpy as np

from ..linalg import np_conserved as npc
from ..linalg.krylov_based import LanczosEvolution
from ..linalg.truncation import TruncationError, svd_theta
from .dmrg import TwoSiteDMRGEngine, SingleSiteDMRGEngine
from .mps_common import OneSiteH, ZeroSiteH, IdentityEnvRejected

logger = logging.getLogger(__name__)

__all__ = ['TwoSiteTDVPEngine', 'SingleSiteTDVPEngine']


class _TDVPBase:
    """What the two TDVP engines share (reference tdvp.py:58 and `TimeEvolutionAlgorithm`, algorithm.py:341); mixed into a
    DMRG engine, whose sweep and environment code it reuses."""

    def __init__(self, psi, model, options):
        if not getattr(psi, 'finite', True) or getattr(psi, 'bc', 'finite') != 'finite':
            raise NotImplementedError('Only finite TDVP is implemented')
        options = dict(options or {})
        if options.get('time_dependent_H', False):
            raise NotImplementedError('TDVP with a time-dependent Hamiltonian')
        if int(dict(options.get('Krylov_params', None) or {}).get('expansion_dim', 0)) > 0:
            raise NotImplementedError("Krylov subspace expansion (Krylov_params['expansion_dim'] > 0)")
        if getattr(model.H_MPO, 'explicit_plus_hc', False):
            raise NotImplementedError('TDVP with an MPO with explicit_plus_hc')
        super().__init__(psi, model, options)
        self.evolved_time = self.options.get('start_time', 0.)
        self.trunc_err = self.options.get('start_trunc_err', TruncationError())
        self.dt = None

    @property
    def S_inv_cutoff(self):
        """Reference mps_common.py:161."""
        return 1.e-8 if any(isinstance(S, npc.Array) for S in self.psi._S) else 1.e-15

    def run(self):
        """Evolve by ``N_steps`` steps of ``dt`` (reference algorithm.py:394); returns `psi`."""
        self.run_evolution(int(self.options.get('N_steps', 1)), self.options.get('dt', 0.1))
        return self.psi

    def run_evolution(self, N_steps, dt):
        """Reference algorithm.py:425: real-time evolution keeps ``psi.norm`` unless ``preserve_norm`` is False."""
        preserve_norm = self.options.get('preserve_norm', None)
        if preserve_norm is None:
            preserve_norm = not np.iscomplex(dt)
        old_norm = self.psi.norm
        trunc_err = self.evolve(N_steps, dt)
        self.trunc_err = self.trunc_err + trunc_err
        if preserve_norm:
            self.psi.norm = old_norm

    def evolve(self, N_steps, dt):
        """`N_steps` sweeps of ``dt`` (reference tdvp.py:211); returns the accumulated TruncationError."""
        max_dt = self.options.get('max_dt', 1.)
        if max_dt is None:
            if abs(dt) > 1.:
                logger.warning('dt > ``max_dt`` is unreasonably large for TDVP.')
        elif not abs(dt) <= max_dt:
            raise ValueError('dt > ``max_dt`` is unreasonably large for TDVP.')
        self.dt = dt
        trunc_err = TruncationError()
        for _ in range(N_steps):
            self.sweep()
            for eps in self.trunc_err_list:
                trunc_err = trunc_err + TruncationError(eps, 1. - 2. * eps)
        self.evolved_time = self.evolved_time + N_steps * self.dt
        return trunc_err

    def _krylov_evolve(self, H, theta, dt):
        """``expm(dt H) theta`` by :class:`LanczosEvolution` (reference tdvp.py:132).  A real `theta` with a complex `H` is
        promoted first (the Krylov vectors then stay on the device-scalar route); the deferred test of the identity
        shortcut of the split-order matvec restarts the evolution without it, as in DMRG."""
        if not self.lanczos_params.get('hermitian', True):
            raise NotImplementedError("lanczos_params['hermitian'] = False: non-hermitian evolution needs the reference's "
                                      "ArnoldiEvolution, which the engine does not provide")
        normalize = self.lanczos_params.get('normalize', None)
        if np.dtype(H.dtype).kind == 'c' and np.dtype(theta.dtype).kind != 'c':
            theta = theta.astype(np.complex128)
        lz = LanczosEvolution(H, theta, self.lanczos_params)
        try:
            theta_new, N = lz.run(dt, normalize=normalize)
        except IdentityEnvRejected:
            lz = LanczosEvolution(H, theta, self.lanczos_params)
            theta_new, N = lz.run(dt, normalize=normalize)
        n2 = getattr(lz, '_result_norm2_dev', None)
        if n2 is not None:                   # conditioning test of the result, read at the end of the sweep
            self._pending_scalars.append(('norm2', None, n2))
        return theta_new, N

    def update_env(self, **update_data):
        """Nothing: the environments are updated inside :meth:`update_local` (reference tdvp.py:304)."""


class TwoSiteTDVPEngine(_TDVPBase, TwoSiteDMRGEngine):
    """Two-site TDVP (reference tdvp.py:233): the two-site wave function evolves forward by ``dt/2``, is split by a
    truncated SVD, and the site the sweep moves to evolves backward by ``dt/2``; the last bond of the right sweep
    evolves by ``dt`` at once."""

    def get_sweep_schedule(self):
        """Reference tdvp.py:253."""
        L = self.psi.L
        i0s = list(range(0, L - 2)) + list(range(L - 2, -1, -1))
        move_right = [True] * (L - 2) + [False] * (L - 2) + [None]
        update_LP_RP = [[True, False]] * (L - 2) + [[False, True]] * (L - 2) + [[False, False]]
        return zip(i0s, move_right, update_LP_RP)

    def update_local(self, theta, optimize=True):
        """Reference tdvp.py:264."""
        i0, L = self.i0, self.psi.L
        dt = -0.5j * self.dt
        if i0 == L - 2:
            dt = 2. * dt                     # instead of updating the last pair of sites twice, we double the time
        theta, N = self._krylov_evolve(self.eff_H, theta, dt)
        theta = self.prepare_svd(theta)
        qtotal_i0 = self.psi.get_B(i0, form=None).qtotal
        U, S, VH, err, renorm = svd_theta(theta, self.trunc_params, qtotal_LR=[qtotal_i0, None],
                                          inner_labels=['vR', 'vL'])
        self.psi.norm *= renorm
        self.psi.set_B(i0, U.split_legs(['(vL.p0)']).replace_label('p0', 'p'), form='A')
        self.psi.set_B(i0 + 1, VH.split_legs(['(p1.vR)']).replace_label('p1', 'p'), form='B')
        self.psi.set_SR(i0, S)
        U.ireplace_label('(vL.p0)', '(vL.p)')            # the labels the environment update of the engine reads
        VH.ireplace_label('(p1.vR)', '(p.vR)')
        update_data = {'err': err, 'N': N, 'U': U, 'VH': VH}
        TwoSiteDMRGEngine.update_env(self, **update_data)  # needed by the one-site step
        if self.move_right:
            self.one_site_update(i0 + 1, 0.5j * self.dt)
        elif self.move_right is False:
            self.one_site_update(i0, 0.5j * self.dt)
        return update_data

    def one_site_update(self, i, dt):
        """Backward evolution of site `i` (reference tdvp.py:308)."""
        H1 = OneSiteH(self.env, i, combine=False)
        theta = H1.combine_theta(self.psi.get_theta(i, n=1, cutoff=self.S_inv_cutoff))
        theta, _ = self._krylov_evolve(H1, theta, dt)
        self.psi.set_B(i, theta.replace_label('p0', 'p'), form='Th')

    def post_update_local(self, err, **update_data):
        self.trunc_err_list.append(err.eps)


class SingleSiteTDVPEngine(_TDVPBase, SingleSiteDMRGEngine):
    """Single-site TDVP (reference tdvp.py:318): one site evolves forward by ``dt/2``, is split by an SVD without
    truncation, and the bond matrix evolves backward by ``dt/2`` under :class:`ZeroSiteH`; bond dimensions do not
    grow."""

    def get_sweep_schedule(self):
        """Reference tdvp.py:335."""
        L = self.psi.L
        i0s = list(range(0, L - 1)) + list(range(L - 1, -1, -1))
        move_right = [True] * (L - 1) + [False] * (L - 1) + [None]
        update_LP_RP = [[True, False]] * (L - 1) + [[False, True]] * (L - 1) + [[False, False]]
        return zip(i0s, move_right, update_LP_RP)

    def update_local(self, theta, optimize=True):
        """Reference tdvp.py:346."""
        i0, L = self.i0, self.psi.L
        dt = -0.5j * self.dt
        if i0 == L - 1:
            dt = 2. * dt                     # instead of updating the last site twice, we double the time
        theta, _ = self._krylov_evolve(self.eff_H, theta, dt)
        if self.move_right:
            self.right_moving_update(i0, theta)
        else:                                # also the last update of the sweep (move_right None)
            self.left_moving_update(i0, theta)
        return {}

    def right_moving_update(self, i0, theta):
        """Reference tdvp.py:364."""
        if self.combine:
            theta.itranspose(['(vL.p0)', 'vR'])
        else:
            theta = theta.combine_legs(['vL', 'p0'], qconj=+1, new_axes=0)
        U, S, VH = npc.svd(theta, qtotal_LR=[theta.qtotal, None], inner_labels=['vR', 'vL'])
        renorm = np.linalg.norm(S)
        S = S / renorm
        self.psi.norm *= renorm
        self.psi.set_B(i0, U.split_legs(['(vL.p0)']).replace_label('p0', 'p'), form='A')
        self.psi.set_SR(i0, S)
        TwoSiteDMRGEngine.update_env(self, U=U.replace_label('(vL.p0)', '(vL.p)'))
        theta = self.zero_site_update(i0 + 1, VH.scale_axis(S, 'vL'), 0.5j * self.dt)
        next_B = self.psi.get_B(i0 + 1, form='B')
        self.psi.set_B(i0 + 1, npc.tensordot(theta, next_B, axes=['vR', 'vL']), form='Th')

    def left_moving_update(self, i0, theta):
        """Reference tdvp.py:386."""
        if self.combine:
            theta.itranspose(['vL', '(p0.vR)'])
        else:
            theta = theta.combine_legs(['p0', 'vR'], qconj=-1, new_axes=1)
        U, S, VH = npc.svd(theta, qtotal_LR=[None, theta.qtotal], inner_labels=['vR', 'vL'])
        renorm = np.linalg.norm(S)
        S = S / renorm
        self.psi.norm *= renorm
        if i0 == 0:
            assert U.shape == (1, 1)
            u = U.to_ndarray()[0, 0]         # just a global phase, but better keep it
            VH = VH * (complex(u) if np.iscomplexobj(u) else float(u))
        self.psi.set_B(i0, VH.split_legs(['(p0.vR)']).replace_label('p0', 'p'), form='B')
        self.psi.set_SL(i0, S)
        if i0 != 0:
            TwoSiteDMRGEngine.update_env(self, VH=VH.replace_label('(p0.vR)', '(p.vR)'))
            theta = self.zero_site_update(i0, U.scale_axis(S, 'vR'), 0.5j * self.dt)
            next_A = self.psi.get_B(i0 - 1, form='A')
            # the Schmidt values left of i0 stay those of the SVD above, as in the reference
            self.psi.set_B(i0 - 1, npc.tensordot(next_A, theta, axes=['vR', 'vL']), form='Th')

    def zero_site_update(self, i, theta, dt):
        """Backward evolution of the bond matrix left of site `i` (reference tdvp.py:419)."""
        theta, _ = self._krylov_evolve(ZeroSiteH(self.env, i), theta, dt)
        return theta

    def post_update_local(self, **update_data):
        self.trunc_err_list.append(0.)
