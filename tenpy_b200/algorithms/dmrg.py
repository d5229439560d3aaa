"""Two-site DMRG on the H100-native tensor engine.

Host-side mirror of the reference driver ``tenpy/algorithms/dmrg.py`` (`run` :63, `DMRGEngine` :112,
`TwoSiteDMRGEngine` :846) and of the sweep logic it inherits from ``mps_common.Sweep`` (:60; `sweep` :345,
`get_sweep_schedule` :419, `prepare_update_local` :498, `update_env` :569) and `IterativeSweeps.run`
(:796).  Same options (``trunc_params``, ``lanczos_params``, ``combine``, ``mixer``, ``mixer_params``,
``chi_list``, ``max_E_err``, ``max_S_err``, ``min_sweeps``, ``max_sweeps``, ``N_sweeps_check``), same update
order, same statistics keys.  Each bond update is: effective-H matvecs inside Lanczos (grouped FP64
tensor-core GEMMs), batched block SVD, environment update -- all on the device; the host only steers.
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import logging
import time

import numpy as np

from .. import backend
from ..linalg import np_conserved as npc
from ..linalg.krylov_based import LanczosGroundState
from ..linalg.truncation import svd_theta
from ..networks.mpo import MPOEnvironment
from .mps_common import OneSiteH, TwoSiteH, DensityMatrixMixer, SubspaceExpansion, IdentityEnvRejected

logger = logging.getLogger(__name__)


class _PendingOverlap:
    """<theta_guess|theta> left on the device by `diag` (resolved into ``update_stats['ov_change']`` at the end of the sweep)"""
    __slots__ = ('dev',)

    def __init__(self, dev):
        self.dev = dev

__all__ = ['run', 'TwoSiteDMRGEngine', 'SingleSiteDMRGEngine', 'chi_list', 'entropy', 'full_diag_effH']


def entropy(p, n=1):
    """von-Neumann / Renyi entropy of a probability vector (reference tools/math.py:66)."""
    p = np.asarray(p)
    p = p[p > 1.e-30]
    if n == 1:
        return float(-np.inner(np.log(p), p))
    if n == np.inf:
        return float(-np.log(np.max(p)))
    return float(np.log(np.sum(p**n)) / (1. - n))


def chi_list(chi_max, dchi=20, nsweeps=20):
    """Ramp of bond dimensions ``{sweep: chi}`` (reference dmrg.py:1142)."""
    warmup = int(chi_max / dchi)
    if warmup == 0:
        return {0: chi_max}
    res = {}
    for i in range(warmup):
        res[i * nsweeps] = (i + 1) * dchi
    if chi_max > warmup * dchi:
        res[warmup * nsweeps] = chi_max
    return res


def run(psi, model, options):
    """Run DMRG; `psi` is optimised in place (reference dmrg.py:63).  ``options['active_sites']`` (default 2) selects
    :class:`TwoSiteDMRGEngine` or :class:`SingleSiteDMRGEngine`.

    Returns a dict with ``E``, ``shelve``, ``bond_statistics``, ``sweep_statistics``."""
    active_sites = dict(options or {}).get('active_sites', 2)
    if active_sites == 1:
        engine = SingleSiteDMRGEngine(psi, model, options)
    elif active_sites == 2:
        engine = TwoSiteDMRGEngine(psi, model, options)
    else:
        raise ValueError('For DMRG, can only use 1 or 2 active sites, not {0!r}'.format(active_sites))
    E, _ = engine.run()
    return {'E': E, 'shelve': False, 'bond_statistics': engine.update_stats,
            'sweep_statistics': engine.sweep_stats}


def full_diag_effH(effH, theta_guess, keep_sector=True):
    """Exact diagonalisation of a small effective Hamiltonian (reference dmrg.py:1176).

    The matrix is contracted with the same device operations as the matvec and diagonalised by the batched
    Jacobi `eigh` kernel; only the block of the charge sector of `theta_guess` is used."""
    if not keep_sector:
        raise NotImplementedError('keep_sector=False')
    fullH = effH.to_matrix()
    pipe = theta_guess.make_pipe(effH.acts_on, qconj=+1)
    fullH.legs[0].test_equal(pipe)
    qi = pipe.get_qindex_of_charges(theta_guess.qtotal)
    parts = (fullH.re, fullH.im) if isinstance(fullH, npc.ComplexArray) else (fullH,)
    if not any(np.any(part._qdata[:, 0] == qi) for part in parts):
        logger.warning('H is zero in the given block, nothing to diagonalize. We just return the initial state.')
        return 0., theta_guess
    W, V = npc.eigh(fullH)
    sl = pipe.get_slice(qi)
    j = sl.start + int(np.argmin(W[sl]))
    mask = np.zeros(len(W), dtype=bool)
    mask[j] = True
    V.iproject(mask, 1)
    theta = V.squeeze(1)
    theta = theta.split_legs([0]).iset_leg_labels(effH.acts_on)
    return float(W[j]), theta


class TwoSiteDMRGEngine:
    """Engine of the two-site DMRG (reference dmrg.py:846 on top of :112 and mps_common.py:60)."""
    EffectiveH = TwoSiteH
    DefaultMixer = DensityMatrixMixer
    n_optimize = 2

    def __init__(self, psi, model, options):
        self.psi = psi
        self.model = model
        self.options = options = dict(options or {})
        self.finite = True
        self.combine = options.get('combine', True)
        self.trunc_params = dict(options.get('trunc_params', {}))
        self.lanczos_params = dict(options.get('lanczos_params', {}))
        self.chi_list = options.get('chi_list', None)
        self.diag_method = options.get('diag_method', 'default')
        if self.diag_method not in ('default', 'lanczos', 'ED_block'):
            raise NotImplementedError('diag_method ' + repr(self.diag_method))
        self.N_sweeps_check = options.get('N_sweeps_check', 1)
        default_min_sweeps = int(1.5 * self.N_sweeps_check)
        if self.chi_list is not None:
            default_min_sweeps = max(max(self.chi_list.keys()), default_min_sweeps)
        options.setdefault('min_sweeps', default_min_sweeps)
        mixer_params = options.setdefault('mixer_params', {})
        mixer_params.setdefault('amplitude', 1.e-5)       # finite-chain defaults of the reference (dmrg.py:205-212)
        mixer_params.setdefault('decay', 2.)
        mixer_params.setdefault('disable_after', 15)
        self.sweeps = options.get('sweep_0', 0)
        self.time0 = time.time()
        self.mixer = None
        # warm start of the Jacobi SVD from the previous update of the same bond (extension, off by default):
        #   False      : cold start every time (default);
        #   'full'     : rotate theta with the complete previous singular vector bases (keeps 2 (chi d)^2 doubles per bond);
        #   'subspace' : decompose theta inside the span of the previously kept isometry when the part outside is below
        #                the truncation tolerance (truncation.svd_theta); keeps the truncated (U, VH) of every bond.
        ws = options.get('svd_warm_start', False)
        self.svd_warm_start = 'full' if ws is True else ws
        self._svd_guess = {}
        self.env = MPOEnvironment(psi, model.H_MPO, psi)
        self.eff_H = None
        self.i0 = 0
        self.move_right = True
        self.update_LP_RP = (True, False)
        self.E_trunc_list = []
        self.trunc_err_list = []
        self._meas_E_trunc = False
        self._entropy_approx = [None] * psi.L
        self.reset_stats()

    # ------------------------------------------------------------------ statistics
    def reset_stats(self):
        """Reference dmrg.py:492."""
        self.update_stats = {'i0': [], 'age': [], 'E_total': [], 'N_lanczos': [], 'time': [], 'err': [],
                             'E_trunc': [], 'ov_change': []}
        self.sweep_stats = {'sweep': [], 'N_updates': [], 'E': [], 'Delta_E': [], 'S': [], 'Delta_S': [],
                            'max_S': [], 'time': [], 'max_trunc_err': [], 'max_E_trunc': [], 'max_chi': [],
                            'norm_err': []}
        self.shelve = False
        self.time0 = time.time()
        self._pending_scalars = []       # (kind, index, 1-element device tensor): statistics read at the end of a sweep

    # ------------------------------------------------------------------ mixer
    def mixer_activate(self):
        """Reference mps_common.py:653."""
        Mixer_class = self.options.get('mixer', False)
        if not Mixer_class:
            return
        if Mixer_class is True:
            Mixer_class = self.DefaultMixer
        elif isinstance(Mixer_class, str):
            known = {'DensityMatrixMixer': DensityMatrixMixer, 'SubspaceExpansion': SubspaceExpansion}
            if Mixer_class not in known:
                raise ValueError('unknown mixer ' + repr(Mixer_class))
            Mixer_class = known[Mixer_class]
        self.mixer = Mixer_class(dict(self.options.get('mixer_params', {})), self.sweeps)

    def mixer_deactivate(self):
        self.mixer = None

    def mixer_cleanup(self):
        """Bring the 2-D bond matrices a mixer sweep leaves back to diagonal form: ``S = U s V``, `U` and `V` are
        absorbed into the neighbouring tensors and into the stored environments (reference mps_common.py:693)."""
        psi = self.psi
        for i in range(1, psi.L):
            S = psi.get_SL(i)
            if not isinstance(S, npc.Array):
                continue
            U, S, V = npc.svd(S, full_matrices=False, inner_labels=['vR', 'vL'])
            form_L = psi.form[i - 1][1]
            form_R = psi.form[i][0]
            B_L = psi.get_B(i - 1, form=None)
            B_R = psi.get_B(i, form=None)
            if form_L == 0.:
                B_L = npc.tensordot(B_L, U, ['vR', 'vL'])
            elif form_L == 1.:
                B_L = npc.tensordot(B_L, V.conj().replace_labels(['vR*', 'vL*'], ['vL', 'vR']), ['vR', 'vL'])
            else:
                raise RuntimeError('Array S are only supported in A, B, Th or G form.')
            if form_R == 0.:
                B_R = npc.tensordot(V, B_R, ['vR', 'vL'])
            elif form_R == 1.:
                B_R = npc.tensordot(U.conj().replace_labels(['vR*', 'vL*'], ['vL', 'vR']), B_R, ['vR', 'vL'])
            else:
                raise RuntimeError('Array S are only supported in A, B, Th or G form.')
            psi.set_B(i - 1, B_L, form=psi.form[i - 1])
            psi.set_SL(i, S)
            psi.set_B(i, B_R, form=psi.form[i])
            if self.env.has_LP(i):
                LP = self.env.get_LP(i)
                LP = npc.tensordot(LP, U.conj(), ['vR*', 'vL*'])
                LP = npc.tensordot(LP, U, ['vR', 'vL'])
                LP.itranspose(['vR*', 'wR', 'vR'])
                self.env.set_LP(i, LP, age=self.env.get_LP_age(i))
            if self.env.has_RP(i - 1):
                RP = self.env.get_RP(i - 1)
                RP = npc.tensordot(V.conj(), RP, ['vR*', 'vL*'])
                RP = npc.tensordot(V, RP, ['vR', 'vL'])
                RP.itranspose(['vL', 'wL', 'vL*'])
                self.env.set_RP(i - 1, RP, age=self.env.get_RP_age(i - 1))
        self._svd_guess = {}

    # ------------------------------------------------------------------ the run loop (IterativeSweeps.run, :796)
    def run(self):
        self.shelve = False
        self.mixer_activate()                                 # pre_run_initialize (mps_common.py:819)
        while True:
            if self.stopping_criterion(time.time()):
                break
            self.run_iteration()
        self.post_run_cleanup()
        max_trunc = self.options.get('max_trunc_err', 1.e-4)
        if max_trunc is not None and len(self.trunc_err_list) and np.max(self.trunc_err_list) > max_trunc:
            raise ValueError('Maximum truncation error (``max_trunc_err``) exceeded.')   # consistency_check (:810)
        return self.sweep_stats['E'][-1] if len(self.sweep_stats['E']) else np.nan, self.psi

    def stopping_criterion(self, iteration_start_time):
        """Reference mps_common.py:869 (including its ``>`` comparisons: ``max_sweeps + 1`` sweeps are done when
        the run does not converge, and a converged run with an active mixer switches the mixer off and goes on)."""
        min_sweeps = self.options.get('min_sweeps', 1)
        max_sweeps = self.options.get('max_sweeps', 1000)
        max_seconds = 3600 * self.options.get('max_hours', 24 * 365)
        if self.sweeps > max_sweeps:
            return True
        if self.sweeps > min_sweeps and self.is_converged():
            if self.mixer is None:
                return True
            self.mixer_deactivate()
            return False
        if iteration_start_time - self.time0 > max_seconds:
            self.shelve = True
            return True
        return False

    def is_converged(self):
        """Reference dmrg.py:376, verbatim criterion ``|Delta_E / max(E, 1)| < max_E_err and |Delta_S| < max_S_err``
        (note ``max(E, 1)``, not ``max(|E|, 1)``: for negative energies the energy criterion is absolute)."""
        max_E_err = self.options.get('max_E_err', 1.e-8)
        max_S_err = self.options.get('max_S_err', 1.e-5)
        E = self.sweep_stats['E'][-1]
        Delta_E = self.sweep_stats['Delta_E'][-1]
        Delta_S = self.sweep_stats['Delta_S'][-1]
        return abs(Delta_E / max(E, 1.)) < max_E_err and abs(Delta_S) < max_S_err

    def run_iteration(self):
        """`N_sweeps_check` sweeps, adaptive Lanczos tolerances, statistics (reference dmrg.py:219-348)."""
        options = self.options
        p_tol_to_trunc = options.get('P_tol_to_trunc', 0.05)
        if p_tol_to_trunc is not None:
            svd_min = self.trunc_params.get('svd_min', 0.) or 0.
            trunc_cut = self.trunc_params.get('trunc_cut', 0.) or 0.
            p_tol_min = max(1.e-30, svd_min**2 * p_tol_to_trunc, trunc_cut**2 * p_tol_to_trunc)
            p_tol_min = options.get('P_tol_min', p_tol_min)
            p_tol_max = options.get('P_tol_max', 1.e-4)
        e_tol_to_trunc = options.get('E_tol_to_trunc', None)
        if e_tol_to_trunc is not None:
            e_tol_min = options.get('E_tol_min', 5.e-16)
            e_tol_max = options.get('E_tol_max', 1.e-4)
        if len(self.sweep_stats['E']) < 1:
            E_old = np.nan
            S_old = np.mean(self.psi.entanglement_entropy())
        else:
            E_old = self.sweep_stats['E'][-1]
            S_old = self.sweep_stats['S'][-1]
        for _ in range(self.N_sweeps_check - 1):
            self.sweep(meas_E_trunc=False)
        max_trunc_err = self.sweep(meas_E_trunc=True)
        max_E_trunc = np.max(self.E_trunc_list)
        if p_tol_to_trunc is not None and max_trunc_err > p_tol_min:
            self.lanczos_params['P_tol'] = max(p_tol_min, min(p_tol_max, max_trunc_err * p_tol_to_trunc))
        if e_tol_to_trunc is not None and max_E_trunc > e_tol_min:
            self.lanczos_params['E_tol'] = max(e_tol_min, min(e_tol_max, max_E_trunc * e_tol_to_trunc))
        entropy_bonds = self._entropy_approx[1:]
        max_S = max(entropy_bonds)
        S = np.mean(entropy_bonds)
        E = self.update_stats['E_total'][-1]
        norm_err = np.linalg.norm(self.psi.norm_test())
        self.sweep_stats['sweep'].append(self.sweeps)
        self.sweep_stats['N_updates'].append(len(self.update_stats['i0']))
        self.sweep_stats['E'].append(E)
        self.sweep_stats['Delta_E'].append((E - E_old) / self.N_sweeps_check)
        self.sweep_stats['S'].append(S)
        self.sweep_stats['Delta_S'].append((S - S_old) / self.N_sweeps_check)
        self.sweep_stats['max_S'].append(max_S)
        self.sweep_stats['time'].append(time.time() - self.time0)
        self.sweep_stats['max_trunc_err'].append(max_trunc_err)
        self.sweep_stats['max_E_trunc'].append(max_E_trunc)
        self.sweep_stats['max_chi'].append(int(np.max(self.psi.chi)))
        self.sweep_stats['norm_err'].append(norm_err)
        logger.info('sweep %d: E=%.13f S=%.6f chi=%d trunc=%.2e t=%.1fs', self.sweeps, E, S,
                    self.sweep_stats['max_chi'][-1], max_trunc_err, self.sweep_stats['time'][-1])
        return E, self.psi

    def post_run_cleanup(self):
        """Reference dmrg.py:402: `mixer_cleanup`, then `_canonicalize` (:455) -- when the final state violates the
        canonical form by more than ``norm_tol_final`` (a truncating run that is not fully converged), it is
        re-canonicalised with `MPS.canonical_form`, which also refreshes all Schmidt values."""
        self.mixer_cleanup()
        if self.mixer is not None:
            return
        norm_tol = self.options.get('norm_tol', 1.e-5)
        norm_tol_final = self.options.get('norm_tol_final', 1.e-10)
        norm_err = np.linalg.norm(self.psi.norm_test())
        if norm_tol is None or (norm_err < norm_tol and norm_err < norm_tol_final):
            return
        if norm_err > norm_tol:
            logger.warning('final DMRG state not in canonical form up to norm_tol=%.2e: norm_err=%.2e', norm_tol,
                           norm_err)
        if norm_err > norm_tol_final:
            self.psi.canonical_form()
            self.env.clear()
            self._svd_guess = {}

    # ------------------------------------------------------------------ one sweep (mps_common.py:345)
    def get_sweep_schedule(self):
        L, n = self.psi.L, self.n_optimize
        assert L > n
        i0s = list(range(0, L - n)) + list(range(L - n, 0, -1))
        move_right = [True] * (L - n) + [False] * (L - n)
        update_LP_RP = [[True, False]] * (L - n) + [[False, True]] * (L - n)
        return zip(i0s, move_right, update_LP_RP)

    def sweep(self, optimize=True, meas_E_trunc=False):
        """One sweep right and back left (reference mps_common.py:345, dmrg.py:520)."""
        self._meas_E_trunc = meas_E_trunc
        self.E_trunc_list = []
        self.trunc_err_list = []
        if optimize and self.chi_list is not None:
            new_chi_max = self.chi_list.get(self.sweeps, None)
            if new_chi_max is not None:
                self.trunc_params['chi_max'] = new_chi_max
                if self.options.get('chi_list_reactivates_mixer', True):
                    self.mixer_activate()
        for i0, move_right, update_LP_RP in self.get_sweep_schedule():
            self.i0, self.move_right, self.update_LP_RP = i0, move_right, update_LP_RP
            theta = self.prepare_update_local()
            update_data = self.update_local(theta, optimize=optimize)
            self.update_env(**update_data)
            self.post_update_local(**update_data)
            self.free_no_longer_needed_envs()
        self.resolve_pending_scalars()
        if optimize:
            self.sweeps += 1
            if self.mixer is not None:
                mixer = self.mixer.update_amplitude(self.sweeps)
                if mixer is None:
                    self.mixer_deactivate()
                else:
                    self.mixer = mixer
        return np.max(self.trunc_err_list)

    def resolve_pending_scalars(self):
        """read the statistics the bond updates left on the device (one transfer): overlaps -> ``update_stats['ov_change']``,
        norms of the Lanczos results -> the reference's conditioning warning"""
        pend, self._pending_scalars = self._pending_scalars, []
        if not pend:
            return
        import torch
        vals = backend.to_host(torch.cat([t for _, _, t in pend]))
        for (kind, idx, _), v in zip(pend, vals):
            if kind == 'ov':
                self.update_stats['ov_change'][idx] = 1. - abs(float(v))
            elif abs(1. - np.sqrt(v)) > 1.e-5:
                logger.warning('poorly conditioned H matrix in KrylovBased! |psi_0| = %f', np.sqrt(v))

    def prepare_update_local(self):
        """Reference mps_common.py:498."""
        self.eff_H = self.EffectiveH(self.env, self.i0, self.combine, self.move_right,
                                      matvec_order=self.options.get('matvec_order', 'auto'))
        if 'identity_env' in self.options:
            self.eff_H.identity_env = bool(self.options['identity_env'])
        # this engine's Lanczos calls `eff_H.deferred_check()` after its first read-back (and `diag` restarts on rejection)
        self.eff_H.identity_check = self.options.get('identity_check', 'deferred')
        theta = self.psi.get_theta(self.i0, n=self.n_optimize)
        return self.eff_H.combine_theta(theta)

    def update_local(self, theta, optimize=True):
        """Reference dmrg.py:529."""
        i0 = self.i0
        n_opt = self.n_optimize
        age = self.env.get_LP_age(i0) + n_opt + self.env.get_RP_age(i0 + n_opt - 1)
        if optimize:
            E0, theta, N, ov_change = self.diag(theta)
        else:
            E0, N, ov_change = None, 0, 0.
        theta = self.prepare_svd(theta)
        U, S, VH, err, S_approx = self.mixed_svd(theta)
        self._entropy_approx[(i0 + n_opt - 1) % self.psi.L] = entropy(np.asarray(S_approx)**2)
        self.set_B(U, S, VH)
        return {'E0': E0, 'err': err, 'N': N, 'age': age, 'U': U, 'VH': VH, 'ov_change': ov_change}

    def diag(self, theta_guess):
        """Reference dmrg.py:672: Lanczos, or for ``diag_method='default'`` and tiny effective Hamiltonians
        (``N < max_N_for_ED``) the exact diagonalisation of the charge block (`full_diag_effH`)."""
        N = -1
        if self.eff_H.dtype is not np.float64 and not isinstance(theta_guess, npc.ComplexArray):
            theta_guess = theta_guess.astype(np.complex128)       # a real state, a complex Hamiltonian
        if self.diag_method == 'ED_block' or (self.diag_method == 'default' and
                                              self.eff_H.N < self.options.get('max_N_for_ED', 400)):
            E, theta = full_diag_effH(self.eff_H, theta_guess, keep_sector=True)
        else:
            lz = LanczosGroundState(self.eff_H, theta_guess, self.lanczos_params)
            try:
                E, theta, N = lz.run()
            except IdentityEnvRejected:      # the deferred test of the matvec shortcut failed: plain contraction order
                lz = LanczosGroundState(self.eff_H, theta_guess, self.lanczos_params)
                E, theta, N = lz.run()
            n2 = getattr(lz, '_result_norm2_dev', None)
            if n2 is not None:               # conditioning test of the Lanczos result, read at the end of the sweep
                self._pending_scalars.append(('norm2', None, n2))
        # overlap of the new with the old wave function: a statistic only -- computed on the device now, read with all the
        # others at the end of the sweep (no host round trip between the Lanczos result and the SVD)
        if not isinstance(theta, npc.ComplexArray) and not isinstance(theta_guess, npc.ComplexArray) and \
                theta_guess._layout.nblocks and theta_guess._layout.same_blocks(theta._layout) and \
                theta_guess.get_leg_labels() == theta.get_leg_labels() and np.all(theta_guess.qtotal == theta.qtotal):
            lib = backend.get_lib()
            ov = backend.empty(1)
            lib.dot(theta._layout.size, theta_guess._buf, theta._buf, backend.dot_scratch(), ov)
            return E, theta, N, _PendingOverlap(ov)
        ov_change = 1. - abs(npc.inner(theta_guess, theta, 'labels', do_conj=True))
        return E, theta, N, ov_change

    def prepare_svd(self, theta):
        if self.combine:
            return theta
        return theta.combine_legs([['vL', 'p0'], ['p1', 'vR']], new_axes=[0, 1], qconj=[+1, -1])

    def mixed_svd(self, theta):
        """Reference dmrg.py:876."""
        i0 = self.i0
        update_LP, update_RP = self.update_LP_RP
        if self.mixer is None:
            qtotal_i0 = self.psi.get_B(i0, form=None).qtotal
            ws = self.svd_warm_start
            full = [] if ws == 'full' else None
            U, S, VH, err, _ = svd_theta(theta, self.trunc_params, qtotal_LR=[qtotal_i0, None],
                                         inner_labels=['vR', 'vL'],
                                         guess=self._svd_guess.get(i0) if ws == 'full' else None, full_out=full,
                                         subspace=self._svd_guess.get(i0) if ws == 'subspace' else None)
            if full:
                self._svd_guess[i0] = full[0]
            elif ws == 'subspace':
                self._svd_guess[i0] = (U.copy(deep=False), VH.copy(deep=False))
            S_a = S
        else:
            old_BL_qtotal = self.psi.get_B(i0, form=None).qtotal
            qtotal_LR = [old_BL_qtotal, theta.chinfo.make_valid(theta.qtotal - old_BL_qtotal)]
            U, S, VH, err, S_a = self.mixer.mix_and_decompose_2site(engine=self, theta=theta, i0=i0,
                                                                    mix_left=update_LP, mix_right=update_RP,
                                                                    qtotal_LR=qtotal_LR)
        U.ireplace_label('(vL.p0)', '(vL.p)')
        VH.ireplace_label('(p1.vR)', '(p.vR)')
        return U, S, VH, err, S_a

    def _update_env_inds(self):
        """left and right updated site (reference mps_common.py:591)"""
        if self.n_optimize == 2 or self.move_right:
            return self.i0, self.i0 + 1
        return self.i0 - 1, self.i0

    def set_B(self, U, S, VH):
        """Reference dmrg.py:934 / :1112."""
        i_L, i_R = self._update_env_inds()
        B0 = U.split_legs(['(vL.p)'])
        B1 = VH.split_legs(['(p.vR)'])
        self.psi.set_B(i_L, B0, form='A')
        self.psi.set_B(i_R, B1, form='B')
        self.psi.set_SR(i_L, S)

    def update_env(self, **update_data):
        """Reference mps_common.py:569: the parts across the updated bond are dropped, the one needed next is
        recomputed from `LHeff` / `RHeff` (TwoSiteH.update_LP / update_RP)."""
        i_L, i_R = self._update_env_inds()
        self.env.del_LP(i_R)
        self.env.del_RP(i_L)
        update_LP, update_RP = self.update_LP_RP
        if update_LP:
            self.eff_H.update_LP(self.env, i_R, update_data['U'])
        if update_RP:
            self.eff_H.update_RP(self.env, i_L, update_data['VH'])

    def post_update_local(self, E0, age, N, ov_change, err, **update_data):
        """Reference dmrg.py:575."""
        i0 = self.i0
        E_trunc = None
        if self._meas_E_trunc or E0 is None:
            E_trunc = float(np.real(self.env.full_contraction(self._update_env_inds()[0])))   # uses the updated LP / RP
            if E0 is None:
                E0 = E_trunc
            E_trunc = E_trunc - E0
        self.trunc_err_list.append(err.eps)
        self.E_trunc_list.append(E_trunc)
        self.update_stats['i0'].append(i0)
        self.update_stats['age'].append(age)
        self.update_stats['E_total'].append(E0)
        self.update_stats['E_trunc'].append(E_trunc)
        self.update_stats['N_lanczos'].append(N)
        self.update_stats['err'].append(err)
        if isinstance(ov_change, _PendingOverlap):
            self._pending_scalars.append(('ov', len(self.update_stats['ov_change']), ov_change.dev))
            ov_change = np.nan
        self.update_stats['ov_change'].append(ov_change)
        self.update_stats['time'].append(time.time() - self.time0)

    def free_no_longer_needed_envs(self):
        """Reference mps_common.py:614: parts that will be recomputed before their next use are dropped."""
        i_L, i_R = self._update_env_inds()
        update_LP, update_RP = self.update_LP_RP
        if self.n_optimize == 2:
            if update_RP:
                self.env.del_LP(i_L)                          # will update (i0-1, i0) next: LP[i0] is useless
            if update_LP:
                self.env.del_RP(i_R)                          # will update (i0+1, i0+2) next: RP[i0+1] is useless
        else:
            if self.move_right and update_RP:
                self.env.del_LP(i_L)
            elif (self.move_right is False) and update_LP:
                self.env.del_RP(i_R)
        self.eff_H = None


class SingleSiteDMRGEngine(TwoSiteDMRGEngine):
    """Engine of the single-site DMRG (reference dmrg.py:955): one site is optimised at a time, the effective
    Hamiltonian is :class:`~tenpy_b200.algorithms.mps_common.OneSiteH` (``LP--W0--RP``, dense matvec cost
    ``O(D d chi^3)``), `theta` is split by an SVD whose non-isometric factor is absorbed into the next site.

    Mixers: ``None`` (bond dimensions and charge sectors of the initial state cannot grow), the default
    :class:`SubspaceExpansion` (one-site cost), or :class:`DensityMatrixMixer`, which cannot decompose a one-site wave
    function and therefore works on the two-site `theta` (two-site cost for the mixing step, as the reference warns,
    dmrg.py:1128)."""
    EffectiveH = OneSiteH
    DefaultMixer = SubspaceExpansion
    n_optimize = 1

    def prepare_svd(self, theta):
        """`'p'` has to point away from the direction we move in (reference dmrg.py:979)."""
        if self.combine:
            if self.move_right:
                theta.itranspose(['(vL.p0)', 'vR'])
            else:
                theta.itranspose(['vL', '(p0.vR)'])
        else:
            if self.move_right:
                theta = theta.combine_legs(['vL', 'p0'], qconj=+1, new_axes=0)
            else:
                theta = theta.combine_legs(['p0', 'vR'], qconj=-1, new_axes=1)
        return theta

    def mixed_svd(self, theta):
        """Reference dmrg.py:998.  Right move: ``theta -- next_B  ==>  U -- S -- VH``; left move:
        ``next_A -- theta  ==>  U -- S -- VH``; `U` has labels ``'(vL.p)', 'vR'``, `VH` ``'vL', '(p.vR)'``."""
        mixer = self.mixer
        move_right = self.move_right
        update_LP, update_RP = self.update_LP_RP
        psi = self.psi
        if move_right:
            next_B = psi.get_B(self.i0 + 1, form='B').combine_legs(['p', 'vR'], qconj=-1, new_axes=1)
            if update_RP:
                assert psi.form[self.i0 + 1] == (0., 1.)
        else:
            next_A = psi.get_B(self.i0 - 1, form='A').combine_legs(['vL', 'p'], qconj=+1, new_axes=0)
            if update_LP:
                assert psi.form[self.i0 - 1] == (1., 0.)
        if mixer is None:
            qtotal = [theta.qtotal, None] if move_right else [None, theta.qtotal]
            U, S, VH, err, _ = svd_theta(theta, self.trunc_params, qtotal_LR=qtotal, inner_labels=['vR', 'vL'])
            S_a = S
            if move_right:   # VH only truncates: VH . next_B is still right-canonical
                VH = npc.tensordot(VH, next_B, axes=['vR', 'vL'])
                U.ireplace_label('(vL.p0)', '(vL.p)')
            else:
                U = npc.tensordot(next_A, U, axes=['vR', 'vL'])
                VH.ireplace_label('(p0.vR)', '(p.vR)')
        elif getattr(mixer, 'can_decompose_1site', False):
            U, S, VH, err = mixer.mix_and_decompose_1site(engine=self, theta=theta, i0=self.i0, move_right=move_right)
            S_a = S
            if move_right:   # `next_B` is the right-canonical B of the MPS; the expanded VH goes into S (2D)
                S = npc.tensordot(S, VH, axes=['vR', 'vL']) if isinstance(S, npc.Array) else VH.iscale_axis(S, 'vL')
                VH = next_B
                U.ireplace_label('(vL.p0)', '(vL.p)')
            else:
                S = npc.tensordot(U, S, axes=['vR', 'vL']) if isinstance(S, npc.Array) else U.iscale_axis(S, 'vR')
                U = next_A
                VH.ireplace_label('(p0.vR)', '(p.vR)')
        else:                # the mixer works on the two-site theta
            if move_right:
                next_B.ireplace_label('(p.vR)', '(p1.vR)')
                theta = npc.tensordot(theta, next_B, axes=['vR', 'vL'])
                i0 = self.i0
            else:
                next_A.ireplace_label('(vL.p)', '(vL.p0)')
                theta.ireplace_label('(p0.vR)', '(p1.vR)')
                theta = npc.tensordot(next_A, theta, axes=['vR', 'vL'])
                i0 = self.i0 - 1
            qtotal_LR = [psi.get_B(i0, form=None).qtotal, psi.get_B(i0 + 1, form=None).qtotal]
            U, S, VH, err, S_a = mixer.mixed_svd_2site(engine=self, theta=theta, i0=i0, mix_left=update_LP,
                                                       mix_right=update_RP, qtotal_LR=qtotal_LR)
            U.ireplace_label('(vL.p0)', '(vL.p)')
            VH.ireplace_label('(p1.vR)', '(p.vR)')
        return U, S, VH, err, S_a
