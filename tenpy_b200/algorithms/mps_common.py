"""The zero-, one- and two-site effective Hamiltonians and the density-matrix mixer.

Host-side mirror of the reference ``tenpy/algorithms/mps_common.py``: `ZeroSiteH` (:1440), `TwoSiteH` (:1245; `matvec` :1321,
`combine_Heff` :1350, `combine_theta` :1374, `update_LP` :1421, `update_RP` :1430) and
`DensityMatrixMixer` (:1903; `mix_rho` :1972, `svd_from_rho` :2029, `_mix_LR` :1846).  The contraction
sequences are the reference's; each ``npc.tensordot`` is one grouped FP64 tensor-core GEMM launch.
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import numpy as np

from ..linalg import np_conserved as npc
from ..linalg.truncation import truncate

__all__ = ['ZeroSiteH', 'OneSiteH', 'TwoSiteH', 'Mixer', 'DensityMatrixMixer', 'SubspaceExpansion']


def _apply_chain(obj, theta, chain, relabel):
    """Run a contraction recipe: `chain` = sequence of ``(side, attribute, axes_of_tensor, axes_of_theta)``; ``side``
    'L' contracts ``tensor . theta``, 'R' contracts ``theta . tensor``; `relabel` = (old, new) bra -> ket labels.
    Every step is one grouped GEMM launch (plus block transpositions where the leg order requires them)."""
    for side, attr, ax_t, ax_th in chain:
        tensor = getattr(obj, attr)
        theta = npc.tensordot(tensor, theta, axes=[ax_t, ax_th]) if side == 'L' else \
            npc.tensordot(theta, tensor, axes=[ax_th, ax_t])
    return theta.ireplace_labels(*relabel)


# contraction recipes of the effective Hamiltonians, keyed like the branches of the reference's `matvec` methods
# (mps_common.py:1118-1151 one site, :1321-1348 two sites)
_ONE_SITE_CHAINS = {
    ('combined', True): ([('L', 'LHeff', ['(vR.p0*)'], ['(vL.p0)']), ('R', 'RP', ['wL', 'vL'], ['wR', 'vR'])],
                         (['(vR*.p0)', 'vL*'], ['(vL.p0)', 'vR'])),
    ('combined', False): ([('R', 'RHeff', ['(p0*.vL)'], ['(p0.vR)']), ('L', 'LP', ['vR', 'wR'], ['vL', 'wL'])],
                          (['vR*', '(p0.vL*)'], ['vL', '(p0.vR)'])),
    ('plain', None): ([('L', 'LP', ['vR'], ['vL']), ('L', 'W0', ['wL', 'p0*'], ['wR', 'p0']),
                       ('R', 'RP', ['wL', 'vL'], ['wR', 'vR'])], (['vR*', 'vL*'], ['vL', 'vR'])),
}
_TWO_SITE_CHAINS = {
    'combined': ([('L', 'LHeff', ['(vR.p0*)'], ['(vL.p0)']), ('R', 'RHeff', ['wL', '(p1*.vL)'], ['wR', '(p1.vR)'])],
                 (['(vR*.p0)', '(p1.vL*)'], ['(vL.p0)', '(p1.vR)'])),
    'plain': ([('L', 'LP', ['vR'], ['vL']), ('L', 'W0', ['wL', 'p0*'], ['wR', 'p0']),
               ('R', 'W1', ['wL', 'p1*'], ['wR', 'p1']), ('R', 'RP', ['wL', 'vL'], ['wR', 'vR'])],
              (['vR*', 'vL*'], ['vL', 'vR'])),
}


def _is_complex(x):
    return np.dtype(x.dtype).kind == 'c'


_EYE_CACHE = {}


def _cached_eye(comp):
    """identity Array with the legs of the square 2D Array `comp`, kept on the device per leg structure (all saturated
    bonds of a chain share one); avoids building and uploading a dense identity for every bond"""
    key = (comp.legs[0].content_key(), tuple(comp.get_leg_labels()))
    eye = _EYE_CACHE.get(key)
    if eye is None or eye._buf is None or eye._buf.device != comp._buf.device:
        if len(_EYE_CACHE) > 64:
            _EYE_CACHE.clear()
        eye = _EYE_CACHE[key] = npc.eye_like(comp, 0, labels=comp.get_leg_labels())
    return eye


class OneSiteH:
    r"""Effective Hamiltonian ``LP--W0--RP`` acting on the one-site wave function (reference mps_common.py:1040).

    With ``combine=True`` only the side we move away from is combined: `LHeff` (``'(vR*.p0)', 'wR', '(vR.p0*)'``)
    for a right move, `RHeff` (``'wL', '(p0*.vL)', '(p0.vL*)'``) for a left move; `theta` then has the labels
    ``'(vL.p0)', 'vR'`` or ``'vL', '(p0.vR)'``."""
    length = 1
    acts_on = ['vL', 'p0', 'vR']

    def __init__(self, env, i0, combine=False, move_right=True, matvec_order=None):
        self.i0 = i0
        self.LP = env.get_LP(i0)
        self.RP = env.get_RP(i0)
        self.W0 = env.H.get_W(i0).replace_labels(['p', 'p*'], ['p0', 'p0*'])
        self.dtype = env.H.dtype
        self.combine = combine
        self.move_right = move_right
        self.N = self.LP.get_leg('vR').ind_len * self.W0.get_leg('p0').ind_len * self.RP.get_leg('vL').ind_len
        if combine:
            self.combine_Heff(env)

    def matvec(self, theta):
        """Apply the effective Hamiltonian to `theta` (reference mps_common.py:1118)."""
        key = ('combined', bool(self.move_right)) if self.combine else ('plain', None)
        chain, relabel = _ONE_SITE_CHAINS[key]
        return _apply_chain(self, theta, chain, relabel).itranspose(theta.get_leg_labels())

    def combine_Heff(self, env):
        """Reference mps_common.py:1152."""
        if self.move_right:
            self.LHeff = env._contract_LHeff(self.i0, 'p0')
            self.pipeL = self.LHeff.get_leg('(vR*.p0)')
            self.acts_on = ['(vL.p0)', 'vR']
        else:
            self.RHeff = env._contract_RHeff(self.i0, 'p0')
            self.pipeR = self.RHeff.get_leg('(p0.vL*)')
            self.acts_on = ['vL', '(p0.vR)']

    def combine_theta(self, theta):
        """Reference mps_common.py:1173."""
        if self.combine:
            if self.move_right:
                theta = theta.combine_legs(['vL', 'p0'], pipes=self.pipeL)
            else:
                theta = theta.combine_legs(['p0', 'vR'], pipes=self.pipeR)
        return theta.itranspose(self.acts_on)

    def to_matrix(self):
        """Contract `self` to a 2D Array (reference mps_common.py:1193)."""
        if self.combine:
            if self.move_right:
                contr = npc.tensordot(self.LHeff, self.RP, axes=['wR', 'wL'])
                contr = contr.combine_legs([['(vR*.p0)', 'vL*'], ['(vR.p0*)', 'vL']], qconj=[+1, -1])
            else:
                contr = npc.tensordot(self.LP, self.RHeff, axes=['wR', 'wL'])
                contr = contr.combine_legs([['vR*', '(p0.vL*)'], ['vR', '(p0*.vL)']], qconj=[+1, -1])
        else:
            contr = npc.tensordot(self.LP, self.W0, axes=['wR', 'wL'])
            contr = npc.tensordot(contr, self.RP, axes=['wR', 'wL'])
            contr = contr.combine_legs([['vR*', 'p0', 'vL*'], ['vR', 'p0*', 'vL']], qconj=[+1, -1])
        return contr

    def update_LP(self, env, i, U=None):
        """Reference mps_common.py:1226."""
        if self.combine and self.move_right:
            assert i == self.i0 + 1
            LP = npc.tensordot(self.LHeff, U, axes=['(vR.p0*)', '(vL.p)'])
            LP = npc.tensordot(U.conj(), LP, axes=['(vL*.p*)', '(vR*.p0)'])
            env.set_LP(i, LP, age=env.get_LP_age(i - 1) + 1)
        else:
            env.get_LP(i, store=True)

    def update_RP(self, env, i, VH=None):
        """Reference mps_common.py:1235."""
        if self.combine and (self.move_right is False):
            assert i == self.i0 - 1
            RP = npc.tensordot(VH, self.RHeff, axes=['(p.vR)', '(p0*.vL)'])
            RP = npc.tensordot(RP, VH.conj(), axes=['(p0.vL*)', '(p*.vR*)'])
            env.set_RP(i, RP, age=env.get_RP_age(i + 1) + 1)
        else:
            env.get_RP(i, store=True)


class ZeroSiteH:
    r"""Effective Hamiltonian ``LP--RP`` acting on the bond matrix left of site `i0` (reference mps_common.py:1440): the
    backward step of the single-site TDVP.  `theta` has the labels ``'vL', 'vR'``."""
    length = 0
    acts_on = ['vL', 'vR']

    def __init__(self, env, i0):
        self.i0 = i0
        self.LP = env.get_LP(i0)
        self.RP = env.get_RP(i0 - 1)
        self.dtype = env.H.dtype
        self.N = self.LP.get_leg('vR').ind_len * self.RP.get_leg('vL').ind_len

    def matvec(self, theta):
        """``LP . theta . RP`` (reference mps_common.py:1497)."""
        labels = theta.get_leg_labels()
        theta = npc.tensordot(self.LP, theta, axes=['vR', 'vL'])
        theta = npc.tensordot(theta, self.RP, axes=[['wR', 'vR'], ['wL', 'vL']])
        theta.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
        return theta.itranspose(labels)

    def to_matrix(self):
        """Contract `self` to a 2D Array (small systems only; reference mps_common.py:1518)."""
        contr = npc.tensordot(self.LP, self.RP, axes=['wR', 'wL'])
        return contr.combine_legs([['vR*', 'vL*'], ['vR', 'vL']], qconj=[+1, -1])


def _get_LHeff(env, i, eff_H):
    """`LHeff` with ``p0`` labels on site `i`, reusing the one of `eff_H` if it fits (reference :1885)."""
    if i == eff_H.i0 and hasattr(eff_H, 'LHeff'):
        return eff_H.LHeff
    return env._contract_LHeff(i)


def _mv_dot(a, b, axes, _out=None):
    """`npc.tensordot` for the large products inside an effective-H matvec: on the int8 tensor path with the slice count
    of the Lanczos iteration (``npc.OZAKI['slices_matvec']``, error ~1e-14 relative to (|A||B|)_ij per product)"""
    return npc.tensordot(a, b, axes=axes, _out=_out, _oz_slices=npc.OZAKI['slices_matvec'])


def _get_RHeff(env, i, eff_H):
    """`RHeff` with ``p1`` labels on site `i`, reusing the one of `eff_H` if it fits (reference :1893)."""
    if i == eff_H.i0 + eff_H.length - 1 and hasattr(eff_H, 'RHeff'):
        if eff_H.length == 1:
            return eff_H.RHeff.replace_labels(['(p0.vL*)', '(p0*.vL)'], ['(p1.vL*)', '(p1*.vL)'])
        return eff_H.RHeff
    return env._contract_RHeff(i)


_DENSE_PLANS = {}


def _dense_plan(m, n, k):
    """the grouped-GEMM plan of one dense product (m x k) . (k x n) at offset 0 of raw buffers, kept per shape"""
    from .. import backend
    lib = backend.get_lib()
    hit = _DENSE_PLANS.get((m, n, k))
    if hit is None or hit[0] is not lib:
        if len(_DENSE_PLANS) > 64:
            _DENSE_PLANS.clear()
        q = np.zeros((1, 2), np.int64)
        hit = _DENSE_PLANS[(m, n, k)] = (lib, lib.tdot_plan(q, q, 1, [m], [k], [0], [k], [n], [0]))
    return hit[1]


def _real_embedding(a):
    """the real 2x2 embedding ``[[Ar, -Ai], [Ai, Ar]]`` (row-major, 2m x 2k) of the one-block tensor `a` (real or complex)
    read as the matrix [(leg 0, leg 1), leg 2]"""
    from .. import backend
    lay, planes = npc._planes(a)
    m, k = a.shape[0] * a.shape[1], a.shape[2]
    o = int(lay.offsets[0])
    ar = planes[0][o:o + m * k].view(m, k)
    E = backend.empty(4 * m * k) if len(planes) == 2 else backend.zeros(4 * m * k)
    Ev = E.view(2, m, 2, k)
    Ev[0, :, 0].copy_(ar)
    Ev[1, :, 1].copy_(ar)
    if len(planes) == 2:
        ai = planes[1][o:o + m * k]
        Ev[1, :, 0].copy_(ai.view(m, k))
        neg = ai.clone()
        backend.get_lib().scal(m * k, -1., neg)
        Ev[0, :, 1].copy_(neg.view(m, k))
    return E


def _stacked_planes(a):
    """the planes of the one-block tensor `a` (real or complex) stacked in one buffer ``[Ar; Ai]``"""
    from .. import backend
    lay, planes = npc._planes(a)
    n, o = int(lay.sizes[0]), int(lay.offsets[0])
    S = backend.empty(2 * n) if len(planes) == 2 else backend.zeros(2 * n)
    for j, p in enumerate(planes):
        S[j * n:(j + 1) * n].copy_(p[o:o + n])
    return S


class IdentityEnvRejected(Exception):
    """raised by `SplitOrderMatvec.deferred_check` when the environments turn out not to have identity components: the
    caller restarts its iteration, the effective Hamiltonian has switched the shortcut off"""


class SplitOrderMatvec:
    r"""The split-order routes of the two-site matvec, shared by the engine's `TwoSiteH` and the drop-in effective
    Hamiltonian of the reference's engine (:func:`tenpy_b200.dropin.fast_two_site_engine`).  The class using it provides
    ``i0, LP, RP, W0, W1, combine, pipeL, pipeR`` (as the reference's ``TwoSiteH`` with ``combine=True``) and ``_H_mpo``
    (the MPO), and sends `matvec` to :meth:`_matvec_split` where :meth:`_use_split` says so.

    `matvec_order` (extension; same result, fewer flops): ``'combined'`` is the reference's sequence
    ``LHeff . theta . RHeff``, dense cost :math:`4 D d^3 \chi^3` flops.  ``'split'`` keeps the combined interface (theta
    with the pipes ``(vL.p0)``, ``(p1.vR)``; `LHeff`/`RHeff` are still formed for the environment update and the mixer)
    but applies ``LP``, the two-site MPO tensor ``W0.W1`` and ``RP`` one after the other to the split theta -- the
    contraction order of the reference's ``combine=False`` branch (:1340), dense cost :math:`4 D d^2 \chi^3 + O(\chi^2)`,
    i.e. `d` times fewer flops in the two large GEMMs.  ``'auto'`` (default) takes ``'split'`` when the largest block of
    theta has at least ``SPLIT_MIN_BLOCK`` elements (compute-bound regime) and ``'combined'`` for small ragged blocks,
    where the number of launches decides.

    The shapes alone choose how ``W0.W1`` is applied: to dense tensors (one block) with ``K = D d^2 <= 32`` contracted
    rows (``K1 + K2 = (D-1) d^2 + d^2`` without the identity components) by the streaming kernel b200_mid_contract(2)_f64,
    which keeps the layout; otherwise by `npc.tensordot` (two block transpositions and a skinny GEMM).

    Complex theta and MPOs take the same routes with the same rule for ``'auto'`` (the largest block of either plane of
    theta): with charges `npc.tensordot` composes each complex product of real ones; dense, with the packed complex
    Krylov vector, the replayed kernel sequence uses b200_mid_contract2_z (see :meth:`_dense_z_run`)."""
    SPLIT_MIN_BLOCK = 1 << 20
    matvec_order = 'auto'
    # skip the identity components of the environments in the split-order matvec (see _identity_env_setup): host logic on
    # the GPU-verified kernels, results checked against the reference goldens; engine option `identity_env` switches it off
    identity_env = True
    # 'immediate' (default): the numerical test LP[IdL] = RP[IdR] = 1 costs two blocking reads before the first matvec of
    # the bond; 'deferred': it is evaluated on the device and read back by the caller at its next synchronisation
    # (`deferred_check`; on failure `IdentityEnvRejected` is raised and the caller restarts without the shortcut) -- only
    # for callers that do call `deferred_check` (the DMRG engines set it; their Lanczos checks after its first read-back)
    identity_check = 'immediate'
    stats = {'identity_env_bonds': 0, 'identity_env_rejected': 0}     # diagnostics (how often the shortcut applied)

    # per-instance state, made by the routes on first use
    _W01 = _W01_mat = _RP_t = None                     # W0.W1; plain split order: W0.W1 as a matrix, RP transposed
    _id_env = None                                     # identity shortcut: None until decided, then True / False
    _id_check = None                                   # its pending deferred test
    _LP_rest = _RP_rest = _leg_IdL = _leg_IdR = _W01p = _mask_rest_r = _mpo_cache = None   # see _identity_env_prepare
    _M_id = _N1 = _fused_legs = _RP_rest_t = None      # fused identity route, see _bind_fused_identity
    _dense_recipe = None                               # replayed kernel sequence, see _dense_recipe_bind
    _dense_recipe_off = False
    _dense_z = None                                    # its complex form, see _dense_z_bind
    _dense_z_off = False

    def _use_split(self, theta):
        if self.matvec_order == 'auto':
            # a complex theta: the block tables of its planes (a block of the union of the two is a block of one of them).
            # Complex theta with charges keep the combined order: on the H100 the split order through the composed real
            # products was 0.77x / 0.90x / 0.97x the speed of the combined order for the DM chain (Sz) at chi = 256 / 512 /
            # 1024 (DESIGN.md section 3.3); one-block theta take the dense kernel sequence from SPLIT_MIN_BLOCK on.
            parts = (theta.re, theta.im) if _is_complex(theta) else (theta,)
            sizes = [int(p._layout.sizes.max()) for p in parts if p._layout.nblocks]
            if len(parts) == 2 and max(p._layout.nblocks for p in parts) > 1:
                return False
            return len(sizes) > 0 and max(sizes) >= self.SPLIT_MIN_BLOCK
        return self.matvec_order == 'split'

    def _combine_result(self, out, labels):
        """``out[vL, p0, p1, vR]`` (ours) with the pipes and the label order of theta"""
        out = out.combine_legs([['vL', 'p0'], ['p1', 'vR']], pipes=[self.pipeL, self.pipeR], _view=True)
        return out.itranspose(labels)

    def _matvec_split(self, theta, labels):
        """``LP . theta . (W0 W1) . RP`` on the split legs; interface (labels, pipes) of the combined matvec."""
        if self._W01 is None:
            self._W01 = npc.tensordot(self.W0, self.W1, axes=['wR', 'wL'])   # wL p0 p0* p1 p1* wR  (D^2 d^4 numbers)
        if _is_complex(theta):
            # complex theta: the dense kernel sequence if it applies (_dense_z_run), else the Array-level routes below,
            # whose products npc.tensordot composes of real ones
            out = self._dense_z_run(theta) if self.identity_env and self._id_env is not False else None
            if out is not None:
                return out
        else:
            rec = self._dense_recipe
            if rec is None and not self._dense_recipe_off and self.identity_env:
                rec = self._dense_recipe_from_cache(theta)
            if rec is not None and theta._layout is rec['theta_lay'] and theta._labels == rec['labels']:
                return self._dense_recipe_run(theta, rec)
        th = theta.split_legs(['(vL.p0)', '(p1.vR)'], _view=True)            # vL p0 p1 vR (read only here)
        if self.identity_env and self._id_env is not False:
            try:
                if self._identity_env_setup():
                    return self._matvec_split_identity(th, labels)
            except Exception as e:       # a shortcut must never take the matvec down: plain split order from here on
                import logging
                logging.getLogger(__name__).warning('identity_env shortcut disabled for bond %d: %r', self.i0, e)
                self._id_env = False
        th = _mv_dot(self.LP, th, axes=['vR', 'vL'])                          # vR* wR p0 p1 vR      2 D d^2 chi^3
        fused = self._apply_W01_fused(th)
        if fused is not None:
            th = _mv_dot(fused, self._RP_t, axes=[['wR', 'vR'], ['wL', 'vL']])          # no transposition left
        else:
            th = npc.tensordot(th, self._W01, axes=[['wR', 'p0', 'p1'], ['wL', 'p0*', 'p1*']])  # vR* vR p0 p1 wR
            th = _mv_dot(th, self.RP, axes=[['vR', 'wR'], ['vL', 'wL']])          # vR* p0 p1 vL*   2 D d^2 chi^3
        return self._combine_result(th.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR']), labels)   # th is ours

    def _identity_env_setup(self):
        """In mixed canonical form the component ``wR = IdL`` of `LP` and ``wL = IdR`` of `RP` are identity matrices
        (``<A|1|A>`` / ``<B|1|B>``; the reference contracts them like every other component).  Checked numerically once
        per bond (``|LP[IdL] - 1| <= 1e-11 sqrt(chi)``, same for `RP`); if it holds, the matvec skips these components:
        ``D - 1`` instead of ``D`` large GEMMs on either side.  Prepares `LP` / `RP` without, and ``W0.W1`` with the
        identity components moved to the end of its MPO legs.  Returns False (and remembers it) if not applicable."""
        if self._id_env is not None:
            return self._id_env
        self._id_env = False
        ok = self._identity_env_prepare()
        SplitOrderMatvec.stats['identity_env_bonds' if ok else 'identity_env_rejected'] += 1
        self._id_env = ok
        return ok

    def deferred_check(self):
        """Called by the eigensolver right after one of its own device synchronisations: evaluates the pending test of the
        identity-environment shortcut (free now); raises `IdentityEnvRejected` if it failed."""
        pending = self._id_check
        if not pending:
            return
        self._id_check = None
        from .. import backend
        for out, lim in pending:
            if not backend.read_scalar(out) <= lim:
                self._id_env = False
                self._dense_recipe = self._dense_z = None
                self._dense_recipe_off = True
                SplitOrderMatvec.stats['identity_env_bonds'] -= 1
                SplitOrderMatvec.stats['identity_env_rejected'] += 1
                raise IdentityEnvRejected('environment component differs from the identity')

    def _identity_env_prepare(self):
        H = self._H_mpo
        IdL, IdR = H.get_IdL(self.i0), H.get_IdR(self.i0 + 1)
        if IdL is None or IdR is None or getattr(H, 'explicit_plus_hc', False):
            return False
        LP, RP = self.LP, self.RP
        D_l, D_r = LP.get_leg('wR').ind_len, RP.get_leg('wL').ind_len
        if D_l < 2 or D_r < 2:
            return False
        self._id_check = None
        pending = []
        for part, idx, lab in ((LP, IdL, 'wR'), (RP, IdR, 'wL')):
            comp = part.take_slice(idx, lab)
            if np.any(comp.qtotal != 0):
                return False
            eye = _cached_eye(comp.re if _is_complex(comp) else comp)
            if comp.legs[1].qconj != eye.legs[1].qconj:
                return False
            diff = comp - eye                    # complex: Re LP[IdL] - 1 and Im LP[IdL], both have to vanish
            planes = [p for p in ((diff.re, diff.im) if _is_complex(diff) else (diff,)) if p._layout.nblocks]
            if self.identity_check == 'deferred' and planes:
                # |LP[IdL] - 1|^2 stays on the device; it is read together with the Lanczos scalars (the next unavoidable
                # synchronisation, `deferred_check`), so the set-up costs no round trip of its own
                from .. import backend
                lib = backend.get_lib()
                out = backend.empty(1)
                lib.dot(planes[0]._layout.size, planes[0]._buf, planes[0]._buf, backend.dot_scratch(), out)
                for p in planes[1:]:                                              # + |Im LP[IdL]|^2
                    sq = backend.empty(1)
                    lib.dot(p._layout.size, p._buf, p._buf, backend.dot_scratch(), sq)
                    lib.axpy(1, 1., sq, out)
                pending.append((out, (1.e-11 * np.sqrt(comp.shape[0]))**2))
            elif not npc.norm(diff) <= 1.e-11 * np.sqrt(comp.shape[0]):
                return False
        if pending:
            self._id_check = pending
        only_l, only_r = np.zeros(D_l, bool), np.zeros(D_r, bool)
        only_l[IdL], only_r[IdR] = True, True

        def pieces(arr, label, only):            # (all other components, the identity component with a unit leg)
            rest, one = arr.copy(deep=True), arr.copy(deep=True)
            rest.iproject(~only, label)
            one.iproject(only, label)
            return rest, one

        def rest_of(arr, label, only):           # all other components (one block move) and the unit leg of the identity one
            rest = arr.copy(deep=True)
            rest.iproject(~only, label)
            return rest, arr.get_leg(label).project(only)[2]
        # private copies, constant for the lifetime of this object: their int8 digit planes (npc.OZAKI) are made once
        self._LP_rest, self._leg_IdL = rest_of(LP, 'wR', only_l)
        self._RP_rest, self._leg_IdR = rest_of(RP, 'wL', only_r)
        self._LP_rest._oz_const = self._RP_rest._oz_const = True
        # everything below depends on the MPO and the bond only (not on the state): made once per bond, kept on the MPO
        cache = H.__dict__.setdefault('_b200_two_site_cache', {})
        ent = cache.get(self.i0)
        if ent is None:
            W_rest, W_one = pieces(self._W01, 'wL', only_l)
            W01p = npc.concatenate([W_rest, W_one], axis='wL')                   # wL: [others ..., IdL]
            W_rest, W_one = pieces(W01p, 'wR', only_r)
            ent = cache[self.i0] = {'W01': self._W01, 'W01p': npc.concatenate([W_rest, W_one], axis='wR')}   # wR: [others ..., IdR]
        self._W01, self._W01p = ent['W01'], ent['W01p']
        self._mpo_cache = ent
        self._mask_rest_r = np.arange(D_r) < D_r - 1
        return True

    def _matvec_split_identity(self, th, labels):
        """Split-order matvec without the identity components of the environments: ``T1 = [LP_rest . theta, theta]``,
        ``T2 = (W0 W1) . T1``, ``result = T2[rest] . RP_rest + T2[IdR]``."""
        t1 = _mv_dot(self._LP_rest, th, axes=['vR', 'vL'])                    # vR* wR' p0 p1 vR   2 (D-1) d^2 chi^3
        fused = self._apply_W01_fused_identity(t1, th)
        if fused is not None:
            y_rest, y_id = fused                                             # vR* p0 p1 wR' vR ; vR* p0 p1 vR
            out = _mv_dot(y_rest, self._RP_rest_t, axes=[['wR', 'vR'], ['wL', 'vL']])
            out.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
            out.iadd_prefactor_other(1., y_id.ireplace_label('vR*', 'vL'))
            out = self._combine_result(out, labels)
            self._dense_recipe_record(th, t1, y_rest, y_id, out)
            return out
        th_id = th.add_leg(self._leg_IdL, 0, axis=1, label='wR').ireplace_label('vL', 'vR*')
        t1 = npc.concatenate([t1, th_id], axis='wR')                         # wR: [others ..., IdL]
        t2 = npc.tensordot(t1, self._W01p, axes=[['wR', 'p0', 'p1'], ['wL', 'p0*', 'p1*']])   # vR* vR p0 p1 wR
        views = self._split_t2_views(t2)
        if views is not None:            # no charges: the two components are the two blocks of t2, shared not copied
            t2, direct = views
        else:
            direct = t2.take_slice(len(self._mask_rest_r) - 1, 'wR')        # component IdR: no contraction with RP
            t2.iproject(self._mask_rest_r, 'wR')
        out = _mv_dot(t2, self._RP_rest, axes=[['vR', 'wR'], ['vL', 'wL']])          # vR* p0 p1 vL*  2 (D-1) d^2 chi^3
        out.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
        direct.ireplace_label('vR*', 'vL').itranspose(out.get_leg_labels())
        out.iadd_prefactor_other(1., direct)
        return self._combine_result(out, labels)

    # The dense (no charges, one block per tensor) identity-environment matvec is always the same six kernels: split theta,
    # int8 GEMM with LP_rest, W0 W1 streaming pass, split, int8 GEMM with RP_rest, axpy.  Going through the Array layer
    # (label bookkeeping, leg checks, plan look-ups, result objects) costs ~1 ms of Python per matvec -- as much as the
    # kernels take at chi = 1024 -- so after the first call of a bond the raw sequence is replayed on the buffers.  The
    # geometry of the sequence depends on the MPO and the shapes only: it is kept in the per-bond cache on the MPO, so that
    # later visits of the bond replay it from their first matvec on.
    def _dense_recipe_record(self, th, t1, y_rest, y_id, out):
        """first call of a bond on the fused identity route: record the geometry of its kernels and bind it (`out` is the
        template of the results)"""
        if self._dense_recipe is not None or self._dense_recipe_off:
            return
        arrs = (th, t1, y_rest, y_id, out, self._LP_rest, self._RP_rest_t)
        if any(a._layout.nblocks != 1 for a in arrs) or np.any(out.qtotal != th.qtotal):
            self._dense_recipe_off = True
            return
        chi_l, Dm1, d0, d1, chi_r = t1.shape
        if self._LP_rest.shape != (chi_l, Dm1, chi_l) or self._RP_rest_t.shape != (Dm1, chi_r, chi_r) or \
                out._layout.size != th._layout.size:
            self._dense_recipe_off = True
            return
        plan1 = npc._PLAN_CACHE.get((self._LP_rest._layout.uid, th._layout.uid, 1))
        plan2 = npc._PLAN_CACHE.get((y_rest._layout.uid, self._RP_rest_t._layout.uid, 2))
        if plan1 is None or plan2 is None:
            self._dense_recipe_off = True
            return
        geom = self._mpo_cache['recipe_geom'] = {
            'theta_lay': out._layout, 'labels': list(out._labels), 'plan1': plan1[2], 'plan2': plan2[2],
            'shape_t1': tuple(t1.shape), 'n_t1': int(t1._layout.size), 'n_yr': int(y_rest._layout.size),
            'n_yi': int(y_id._layout.size),
            # buffers whose size is not a multiple of the block alignment carry zero padding (BLAS-1 runs over it)
            'padded': any(a._layout.has_padding for a in (t1, y_rest, y_id, out))}
        self._dense_recipe_bind(geom, out)

    def _dense_recipe_from_cache(self, theta):
        """From the second visit of a bond on (same MPO, same shapes) the kernel sequence is known before the first matvec:
        set up the identity components and bind the recorded geometry to this bond's buffers -- the Array-level route is
        not taken at all.  None if the bond has no recorded geometry (first visit) or anything differs."""
        ent = self._H_mpo.__dict__.get('_b200_two_site_cache', {}).get(self.i0)
        geom = None if ent is None else ent.get('recipe_geom')
        if geom is None or 'M_id' not in ent or theta._layout is not geom['theta_lay'] or theta._labels != geom['labels']:
            return None
        if self._id_env is False or not self._identity_env_setup():
            return None
        chi_l, Dm1, d0, d1, chi_r = geom['shape_t1']
        if self._LP_rest.shape != (chi_l, Dm1, chi_l) or self._RP_rest.get_leg('wL').ind_len != Dm1 or \
                self._LP_rest._layout.nblocks != 1 or self._RP_rest._layout.nblocks != 1:
            return None
        self._bind_fused_identity(ent)
        if self._RP_rest_t.shape != (Dm1, chi_r, chi_r):
            return None
        return self._dense_recipe_bind(geom, theta.copy(deep=False))

    def _dense_recipe_bind(self, geom, template):
        """the replayed kernel sequence of this bond: the recorded geometry, the launch shapes derived from it, and
        `template`, an Array with the layout and labels of the results whose buffer each call replaces"""
        from .. import backend
        chi_l, Dm1, d0, d1, chi_r = geom['shape_t1']
        self._dense_recipe = dict(
            geom, template=template,
            g1=(chi_l * Dm1, d0 * d1 * chi_r, chi_l),                      # (m, n, k) of LP_rest . theta
            g2=(chi_l * d0 * d1, chi_r, Dm1 * chi_r),                      # y_rest . RP_rest
            mid=(Dm1 * d0 * d1, d0 * d1, self._N1, d0 * d1, chi_l, chi_r),
            alloc=backend.zeros if geom['padded'] else backend.empty)
        return self._dense_recipe

    def _dense_recipe_run(self, theta, rec):
        from .. import backend
        lib = backend.get_lib()
        s = npc.OZAKI['slices_matvec']
        alloc = rec['alloc']
        t1 = alloc(rec['n_t1'])
        npc._raw_product(lib, self._LP_rest, theta, rec['g1'], rec['plan1'], t1, s)
        y_r, y_i = alloc(rec['n_yr']), alloc(rec['n_yi'])
        K1, K2, N1, N2, chi_l, chi_r = rec['mid']
        lib.mid_contract2(K1, K2, N1, N2, chi_l, chi_r, self._M_id, t1, theta._buf, y_r, y_i)
        n = rec['theta_lay'].size
        out = alloc(n)
        npc._raw_product(lib, y_r, self._RP_rest_t, rec['g2'], rec['plan2'], out, s)
        lib.axpy(n, 1., y_i, out)
        res = rec['template'].copy(deep=False)
        res._buf = out
        return res

    # The same sequence for a complex theta, on real kernels with doubled dimensions.  theta is the packed Krylov vector
    # of the complex Lanczos (krylov_based._pack): one buffer [theta_r; theta_i], i.e. a (2 chi_l) x (d0 d1 chi_r) matrix.
    #   t1 = [[Lr, -Li], [Li, Lr]] . [theta_r; theta_i]               one DMMA product, result planar [t1_r; t1_i]
    #   Y_emb, Y_id = (W0 W1) . [t1; theta]                             b200_mid_contract2_z: Y_emb = [[Yr, -Yi], [Yi, Yr]]
    #   out = Y_emb . [Rr; Ri]                                          one DMMA product, result planar [out_r; out_i]
    #   out += Y_id                                                     one axpy over both planes
    # The embedding of LP_rest and the stacked planes of RP_rest are constants of the bond (made once, like the
    # int8 digit planes of the real route); the kernel geometry (plans, the complex W0 W1 matrix) is kept in the per-bond
    # cache on the MPO.  Mixed dtypes take the same sequence when theta is complex (a real LP, RP or W0 W1 gets a zero
    # imaginary plane); a real theta with a complex MPO takes the Array-level route (npc.tensordot composes the complex
    # products of real ones), as does every theta that is not a packed, unpadded one-block vector.
    def _dense_z_run(self, theta):
        """the dense complex kernel sequence for `theta`; None if it does not apply (then the Array-level route)"""
        rec = self._dense_z
        if rec is None:
            if self._dense_z_off:
                return None
            try:
                rec = self._dense_z_bind(theta)
            except Exception as e:       # as for the real routes: a shortcut must never take the matvec down
                import logging
                logging.getLogger(__name__).warning('dense complex route disabled for bond %d: %r', self.i0, e)
                rec = None
            if rec is None:
                self._dense_z_off = True
                return None
        if not self._dense_z_fits(theta, rec) or self._id_env is False:
            return None
        from .. import backend
        lib = backend.get_lib()
        s = npc.OZAKI['slices_matvec']
        kbuf = theta._kbuf
        t1 = backend.empty(rec['n_t1'])
        npc._raw_product(lib, rec['E'], kbuf, rec['g1'], rec['plan1'], t1, s)
        y_emb, y_id = backend.empty(rec['n_emb']), backend.empty(2 * rec['n'])
        K1, K2, N1, N2, C1, chi_l, chi_r = rec['mid']
        lib.mid_contract2_z(K1, K2, N1, N2, C1, chi_l, chi_r, rec['M'], t1, kbuf, y_emb, y_id)
        n = rec['n']
        out = backend.empty(2 * n)
        npc._raw_product(lib, y_emb, rec['R'], rec['g2'], rec['plan2'], out, s)
        lib.axpy(2 * n, 1., y_id, out)
        res = npc._from_planes(theta.legs, theta.qtotal, rec['theta_lay'], (out[:n], out[n:]), theta.get_leg_labels())
        res._kbuf = out
        return res

    @staticmethod
    def _dense_z_fits(theta, rec):
        """`theta` is a packed complex vector on the recorded one-block layout: its planes are the two halves of `_kbuf`"""
        kbuf = getattr(theta, '_kbuf', None)
        if kbuf is None or not hasattr(theta, 're') or theta._labels != rec['labels']:
            return False
        lay, n = rec['theta_lay'], rec['n']
        re, im = theta.re, theta.im
        return (re._layout is lay or re._layout.same_blocks(lay)) and (im._layout is lay or im._layout.same_blocks(lay)) \
            and kbuf.numel() == 2 * n and re._buf.data_ptr() == kbuf.data_ptr() and \
            im._buf.data_ptr() == kbuf[n:].data_ptr()

    def _dense_z_bind(self, theta):
        """first complex matvec of the bond: check that the dense sequence applies, make the bond's constants and take the
        kernel geometry from the cache on the MPO (recorded there on the first visit of the bond)"""
        if not hasattr(theta, 're') or getattr(theta, '_kbuf', None) is None:
            return None
        lay = theta.re._layout
        if lay.nblocks != 1 or lay.has_padding or int(lay.offsets[0]) != 0 or \
                theta.get_leg_labels() != ['(vL.p0)', '(p1.vR)']:
            return None
        if self._W01.stored_blocks != 1 or not self._identity_env_setup():
            return None
        rec = {'theta_lay': lay, 'labels': list(theta._labels), 'n': int(lay.size)}
        if not self._dense_z_fits(theta, rec):
            return None
        th = theta.re.split_legs(['(vL.p0)', '(p1.vR)'], _view=True)
        if th._buf.data_ptr() != theta.re._buf.data_ptr() or th.get_leg_labels() != ['vL', 'p0', 'p1', 'vR']:
            return None                  # the pipes are not a plain reshape of the buffer
        chi_l, d0, d1, chi_r = th.shape
        L = self._LP_rest.transpose(['vR*', 'wR', 'vR'])
        R = self._RP_rest.transpose(['wL', 'vL', 'vL*'])
        if L.stored_blocks != 1 or R.stored_blocks != 1:
            return None
        Dl, Dr = L.shape[1], R.shape[0]
        if L.shape != (chi_l, Dl, chi_l) or R.shape != (Dr, chi_r, chi_r):
            return None
        K1, K2, N1, N2 = Dl * d0 * d1, d0 * d1, Dr * d0 * d1, d0 * d1
        if K1 + K2 > 32 or 2 * (N1 + N2) * (K1 + K2) * 8 > 48 * 1024:
            return None
        ent = self._mpo_cache
        geom = ent.get('z_geom')
        shape = (chi_l, Dl, Dr, d0, d1, chi_r)
        if geom is None or geom['shape'] != shape:           # first visit of the bond, or its bond dimensions changed
            geom = ent['z_geom'] = {'shape': shape, 'M': None if geom is None else geom['M']}
            m1, m2, nc = chi_l * Dl, chi_l * d0 * d1, d0 * d1 * chi_r
            geom['g1'], geom['g2'] = (2 * m1, nc, 2 * chi_l), (2 * m2, chi_r, 2 * Dr * chi_r)
            geom['plan1'], geom['plan2'] = _dense_plan(*geom['g1']), _dense_plan(*geom['g2'])
        if geom['M'] is None:
            geom['M'] = self._w01_planes_identity_last()
        rec.update(E=_real_embedding(L), R=_stacked_planes(R), M=geom['M'], g1=geom['g1'], g2=geom['g2'],
                   plan1=geom['plan1'], plan2=geom['plan2'], mid=(K1, K2, N1, N2, Dr, chi_l, chi_r),
                   n_t1=2 * chi_l * Dl * d0 * d1 * chi_r, n_emb=4 * chi_l * d0 * d1 * Dr * chi_r)
        self._dense_z = rec
        return rec

    def _w01_planes_identity_last(self):
        """``W0 W1`` as the planar matrix [Mr | Mi] of [(p0' p1' wR), (wL p0 p1)] with the identity components at the end of
        both MPO index groups (as `M_id` of the real route, :meth:`_apply_W01_fused_identity`)"""
        from .. import backend
        H = self._H_mpo
        IdL, IdR = H.get_IdL(self.i0), H.get_IdR(self.i0 + 1)
        W = self._W01.transpose(['p0', 'p1', 'wR', 'wL', 'p0*', 'p1*']).to_ndarray()
        d0, d1, D_r, D_l = W.shape[0], W.shape[1], W.shape[2], W.shape[3]
        rest_r = [x for x in range(D_r) if x != IdR]
        rest_l = [x for x in range(D_l) if x != IdL]
        rows = np.concatenate([W[:, :, rest_r].reshape(d0 * d1 * len(rest_r), D_l, d0, d1),
                               W[:, :, IdR].reshape(d0 * d1, D_l, d0, d1)], axis=0)
        M = np.concatenate([rows[:, rest_l].reshape(rows.shape[0], -1), rows[:, IdL].reshape(rows.shape[0], -1)], axis=1)
        return backend.to_device(np.concatenate([M.real.reshape(-1), np.imag(M).reshape(-1)]))

    @staticmethod
    def _split_t2_views(t2):
        """``t2`` (legs ``vR*, vR, p0, wR, p1``) with the MPO leg in two sectors [others, IdR] and no other sector structure: the two
        stored blocks ARE the two components.  Returns read-only views ``(t2_rest, direct)`` sharing the packed buffer
        (`direct` without its unit MPO leg), or None if the structure is different (charged tensors) or `t2` is complex
        (then the two components are taken by `take_slice` / `iproject`, plane by plane)."""
        if _is_complex(t2):
            return None
        lay = t2._layout
        ax = t2.get_leg_index('wR')
        leg = t2.legs[ax]
        others = [a for a in range(t2.rank) if a != ax]
        if lay.nblocks != 2 or lay.has_padding or leg.block_number != 2 or np.any(lay.qdata[:, others] != 0) or \
                list(lay.qdata[:, ax]) != [0, 1] or int(lay.shapes[1, ax]) != 1 or \
                any(t2.legs[a].block_number != 1 for a in others):
            return None
        from ..linalg.charges import LegCharge
        chinfo = t2.chinfo
        if np.any(chinfo.make_valid(leg.get_charge(0)) != 0) or np.any(chinfo.make_valid(leg.get_charge(1)) != 0):
            return None
        leg_rest = LegCharge.from_qind(chinfo, leg.slices[:2], leg.charges[:1], leg.qconj)
        n0, n1 = int(lay.sizes[0]), int(lay.sizes[1])
        o0, o1 = int(lay.offsets[0]), int(lay.offsets[1])
        legs_r = list(t2.legs)
        legs_r[ax] = leg_rest
        rest = npc.Array(legs_r, np.float64, t2.qtotal, t2.get_leg_labels())
        lay_r = npc.BlockLayout(np.zeros((1, t2.rank), np.int64), lay.shapes[:1])
        rest._set_blocks(lay_r, t2._buf[o0:o0 + n0])
        direct = npc.Array([t2.legs[a] for a in others], np.float64, t2.qtotal, [t2.get_leg_labels()[a] for a in others])
        lay_d = npc.BlockLayout(np.zeros((1, t2.rank - 1), np.int64), lay.shapes[1:2, others])
        direct._set_blocks(lay_d, t2._buf[o1:o1 + n1])
        return rest, direct

    def _bind_fused_identity(self, ent):
        """bind the per-bond constants of the fused identity route (`ent`: the bond's entry of the cache on the MPO)"""
        self._M_id, self._N1, self._fused_legs = ent['M_id'], ent['N1'], ent['fused_legs']
        self._RP_rest_t = self._RP_rest.transpose(['wL', 'vL', 'vL*'])
        self._RP_rest_t._oz_const = True

    def _apply_W01_fused_identity(self, t1, th):
        """``[Y_rest; Y_IdR] = (W0 W1) . [T1_rest; theta]`` in one streaming pass (b200_mid_contract2_f64): both inputs
        are read once, both outputs come out in the layout their consumer wants.  Dense (one block) only; None if not
        applicable."""
        from .. import backend
        if _is_complex(t1) or _is_complex(th) or _is_complex(self._W01):
            return None                  # complex operands: the dense kernel sequence _dense_z_run, or npc.tensordot
        if t1._layout.nblocks != 1 or th._layout.nblocks != 1 or self._W01._layout.nblocks != 1 or \
                t1.get_leg_labels() != ['vR*', 'wR', 'p0', 'p1', 'vR'] or th.get_leg_labels() != ['vL', 'p0', 'p1', 'vR']:
            return None
        chi_l, Dm1, d0, d1, chi_r = t1.shape
        K1, K2 = Dm1 * d0 * d1, d0 * d1
        if K1 + K2 > 32:
            return None
        if self._M_id is None:
            ent = self._mpo_cache
            if 'M_id' not in ent:
                # (W0 W1) as a matrix [(p0' p1' wR), (wL p0 p1)] with the identity components moved to the end of both
                # index groups; D^2 d^4 model constants, permuted on the host once per bond (and kept on the MPO)
                H = self._H_mpo
                IdL, IdR = H.get_IdL(self.i0), H.get_IdR(self.i0 + 1)
                W = self._W01.transpose(['p0', 'p1', 'wR', 'wL', 'p0*', 'p1*']).to_ndarray()
                D_r, D_l = W.shape[2], W.shape[3]
                rest_r = [x for x in range(D_r) if x != IdR]
                rest_l = [x for x in range(D_l) if x != IdL]
                rows = np.concatenate([W[:, :, rest_r].reshape(d0 * d1 * len(rest_r), D_l, d0, d1),
                                       W[:, :, IdR].reshape(d0 * d1, D_l, d0, d1)], axis=0)
                M = np.concatenate([rows[:, rest_l].reshape(rows.shape[0], -1), rows[:, IdL].reshape(rows.shape[0], -1)],
                                   axis=1)
                ent.update({'M_id': backend.to_device(np.ascontiguousarray(M)), 'N1': d0 * d1 * len(rest_r),
                            'fused_legs': (self._W01.get_leg('p0'), self._W01.get_leg('p1'),
                                           self._RP_rest.get_leg('wL').conj())})
            self._bind_fused_identity(ent)
        N1, N2 = self._N1, K2
        p0leg, p1leg, wleg = self._fused_legs
        legs_r = [t1.legs[0], p0leg, p1leg, wleg, t1.legs[4]]
        legs_i = [t1.legs[0], p0leg, p1leg, t1.legs[4]]
        y_r = npc.Array(legs_r, np.float64, None, ['vR*', 'p0', 'p1', 'wR', 'vR'])
        y_i = npc.Array(legs_i, np.float64, None, ['vR*', 'p0', 'p1', 'vR'])
        lay_r, _ = npc.BlockLayout.from_legs(legs_r, np.zeros((1, 5), np.int64))
        lay_i, _ = npc.BlockLayout.from_legs(legs_i, np.zeros((1, 4), np.int64))
        buf_r = backend.zeros(lay_r.size) if lay_r.has_padding else backend.empty(lay_r.size)
        buf_i = backend.zeros(lay_i.size) if lay_i.has_padding else backend.empty(lay_i.size)
        backend.get_lib().mid_contract2(K1, K2, N1, N2, chi_l, chi_r, self._M_id, t1._buf, th._buf, buf_r, buf_i)
        return y_r._set_blocks(lay_r, buf_r), y_i._set_blocks(lay_i, buf_i)

    def _apply_W01_fused(self, th):
        """``W0.W1`` applied to ``th[vR*, wR, p0, p1, vR]`` in one streaming pass that keeps the layout: the result
        ``[vR*, p0, p1, wR, vR]`` is directly the left operand of the contraction with `RP`.  Dense (one block) only;
        returns None if not applicable."""
        from .. import backend
        W01 = self._W01
        if _is_complex(th) or _is_complex(W01):
            return None                  # complex operands: W0 W1 by npc.tensordot
        if th._layout.nblocks != 1 or W01._layout.nblocks != 1 or th.get_leg_labels() != ['vR*', 'wR', 'p0', 'p1', 'vR']:
            return None
        if self._W01_mat is None:
            self._W01_mat = W01.transpose(['p0', 'p1', 'wR', 'wL', 'p0*', 'p1*'])   # [(p0' p1' wR'), (wL p0 p1)], one block
            self._RP_t = self.RP.transpose(['wL', 'vL', 'vL*'])
        M = self._W01_mat
        chi_l, D, d0, d1, chi_r = th.shape
        K = D * d0 * d1
        N = M.shape[0] * M.shape[1] * M.shape[2]
        if K > 32 or M.size != N * K:
            return None
        legs = [th.legs[0], M.legs[0], M.legs[1], M.legs[2], th.legs[4]]
        res = npc.Array(legs, np.float64, th.chinfo.make_valid(th.qtotal + W01.qtotal),
                        ['vR*', 'p0', 'p1', 'wR', 'vR'])
        lay, _ = npc.BlockLayout.from_legs(legs, np.zeros((1, 5), np.int64))
        buf = backend.zeros(lay.size) if lay.has_padding else backend.empty(lay.size)
        backend.get_lib().mid_contract(K, N, chi_l, chi_r, M._buf, th._buf, buf)
        return res._set_blocks(lay, buf)


class TwoSiteH(SplitOrderMatvec):
    r"""Effective Hamiltonian ``LP--W0--W1--RP`` acting on the two-site wave function (reference :1245).

    With ``combine=True`` (default of the DMRG engine) `LHeff` (labels ``'(vR*.p0)', 'wR', '(vR.p0*)'``)
    and `RHeff` (labels ``'wL', '(p1*.vL)', '(p1.vL*)'``) are formed once per bond and one `matvec` is two
    contractions: ``LHeff . theta`` and ``(..) . RHeff``, dense cost :math:`4 D d^3 \chi^3` flops.  `matvec_order`
    chooses between that order and the split order of :class:`SplitOrderMatvec`."""
    length = 2
    acts_on = ['vL', 'p0', 'p1', 'vR']

    def __init__(self, env, i0, combine=False, move_right=True, matvec_order='auto'):
        if matvec_order not in ('auto', 'combined', 'split'):
            raise ValueError('matvec_order has to be one of auto, combined, split')
        self.matvec_order = matvec_order
        self.i0 = i0
        self.LP = env.get_LP(i0)
        self.RP = env.get_RP(i0 + 1)
        self.W0 = env.H.get_W(i0).replace_labels(['p', 'p*'], ['p0', 'p0*'])
        self.W1 = env.H.get_W(i0 + 1).replace_labels(['p', 'p*'], ['p1', 'p1*'])
        self.dtype = env.H.dtype
        self._H_mpo = env.H
        self.combine = combine
        self.N = (self.LP.get_leg('vR').ind_len * self.W0.get_leg('p0').ind_len *
                  self.W1.get_leg('p1').ind_len * self.RP.get_leg('vL').ind_len)
        if combine:
            self.combine_Heff(env)

    def matvec(self, theta):
        """Apply the effective Hamiltonian to `theta` (reference mps_common.py:1321); real and complex `theta` and MPOs
        alike (the routes of :class:`SplitOrderMatvec`)."""
        labels = theta.get_leg_labels()
        if self.combine and self._use_split(theta):
            return self._matvec_split(theta, labels)
        chain, relabel = _TWO_SITE_CHAINS['combined' if self.combine else 'plain']
        return _apply_chain(self, theta, chain, relabel).itranspose(labels)

    def combine_Heff(self, env, left=True, right=True):
        """Reference mps_common.py:1350.  The pipes are made from the legs right away; the contractions
        ``LHeff = LP.W0`` / ``RHeff = W1.RP`` (each a ``D (d chi)^2`` tensor) are deferred to their first use
        (properties `LHeff` / `RHeff`): with the split-order matvec and no mixer only the side the sweep moves away
        from is ever needed (`update_LP` / `update_RP`)."""
        if left:
            self._LHeff = None
            self.pipeL = npc.LegPipe([self.LP.get_leg('vR*'), self.W0.get_leg('p0')], qconj=+1)
        if right:
            self._RHeff = None
            self.pipeR = npc.LegPipe([self.W1.get_leg('p1'), self.RP.get_leg('vL*')], qconj=-1)
        self.acts_on = ['(vL.p0)', '(p1.vR)']

    @property
    def LHeff(self):
        if not self.combine:
            raise AttributeError('LHeff is only defined for combine=True')
        if self._LHeff is None:
            t = npc.tensordot(self.LP, self.W0, axes=['wR', 'wL'])           # as MPOEnvironment._contract_LHeff
            self._LHeff = t.combine_legs([['vR*', 'p0'], ['vR', 'p0*']], pipes=[self.pipeL, self.pipeL.conj()],
                                         new_axes=[0, 2])
        return self._LHeff

    @LHeff.setter
    def LHeff(self, value):
        self._LHeff = value

    @property
    def RHeff(self):
        if not self.combine:
            raise AttributeError('RHeff is only defined for combine=True')
        if self._RHeff is None:
            t = npc.tensordot(self.W1, self.RP, axes=['wR', 'wL'])           # as MPOEnvironment._contract_RHeff
            self._RHeff = t.combine_legs([['p1', 'vL*'], ['p1*', 'vL']], pipes=[self.pipeR, self.pipeR.conj()],
                                         new_axes=[2, 1])
        return self._RHeff

    @RHeff.setter
    def RHeff(self, value):
        self._RHeff = value

    def combine_theta(self, theta):
        """Reference mps_common.py:1374."""
        if self.combine:
            theta = theta.combine_legs([['vL', 'p0'], ['p1', 'vR']], pipes=[self.pipeL, self.pipeR])
        return theta.itranspose(self.acts_on)

    def to_matrix(self):
        """Contract `self` to a 2D Array (small systems only; reference :1396)."""
        if self.combine:
            contr = npc.tensordot(self.LHeff, self.RHeff, axes=['wR', 'wL'])
            contr = contr.combine_legs([['(vR*.p0)', '(p1.vL*)'], ['(vR.p0*)', '(p1*.vL)']], qconj=[+1, -1])
        else:
            contr = npc.tensordot(self.LP, self.W0, axes=['wR', 'wL'])
            contr = npc.tensordot(contr, self.W1, axes=['wR', 'wL'])
            contr = npc.tensordot(contr, self.RP, axes=['wR', 'wL'])
            contr = contr.combine_legs([['vR*', 'p0', 'p1', 'vL*'], ['vR', 'p0*', 'p1*', 'vL']], qconj=[+1, -1])
        return contr

    def update_LP(self, env, i, U=None):
        """Reference mps_common.py:1421."""
        if self.combine:
            assert i == self.i0 + 1
            LP = npc.tensordot(self.LHeff, U, axes=['(vR.p0*)', '(vL.p)'])
            LP = npc.tensordot(U.conj(), LP, axes=['(vL*.p*)', '(vR*.p0)'])
            env.set_LP(i, LP, age=env.get_LP_age(i - 1) + 1)
        else:
            env.get_LP(i, store=True)

    def update_RP(self, env, i, VH=None):
        """Reference mps_common.py:1430."""
        if self.combine:
            assert i == self.i0
            RP = npc.tensordot(VH, self.RHeff, axes=['(p.vR)', '(p1*.vL)'])
            RP = npc.tensordot(RP, VH.conj(), axes=['(p1.vL*)', '(p*.vR*)'])
            env.set_RP(i, RP, age=env.get_RP_age(i + 1) + 1)
        else:
            env.get_RP(i, store=True)


def _mix_LR(H, i0, amplitude):
    """Diagonal mixing matrices on the MPO bond (reference mps_common.py:1846)."""
    chi_MPO = H.get_W(i0).get_leg('wR').ind_len
    IdL, IdR = H.get_IdL(i0 + 1), H.get_IdR(i0)
    mix_L = np.full((chi_MPO,), amplitude)
    mix_R = np.full((chi_MPO,), amplitude)
    one = 1. if not H.explicit_plus_hc else 0.5
    if IdL is not None:
        mix_L[IdL] = one
        mix_R[IdL] = 0.
    if IdR is not None:
        mix_L[IdR] = 0.
        mix_R[IdR] = one
    return mix_L, mix_R, IdL, IdR, H.explicit_plus_hc


class Mixer:
    """Base class of the mixers (reference mps_common.py:1560): a perturbation of the wave function that lets the
    bond dimension / charge sectors of a bond grow, with an amplitude decaying from sweep to sweep.

    Options `amplitude` (1e-5), `decay` (2.), `disable_after` (15)."""
    can_decompose_1site = False

    def __init__(self, options, sweep_activated=0):
        options = dict(options or {})
        self.amplitude = options.get('amplitude', 1.e-5)
        self.decay = options.get('decay', 2.)
        self.disable_after = options.get('disable_after', 15)
        self.sweep_activated = sweep_activated
        assert self.amplitude <= 1.

    def update_amplitude(self, sweeps):
        """Reference mps_common.py:1626."""
        should_disable = False if self.disable_after is None else \
            sweeps >= self.sweep_activated + self.disable_after
        if self.amplitude is not None and self.decay is not None:
            self.amplitude /= self.decay
            if self.amplitude <= np.finfo('float').eps:
                should_disable = True
        return None if should_disable else self

    def mixed_svd_2site(self, engine, theta, i0, mix_left, mix_right, qtotal_LR=None):
        raise NotImplementedError('{0} does not implement mixed_svd_2site'.format(type(self).__name__))

    def mix_and_decompose_1site(self, engine, theta, i0, move_right):
        raise NotImplementedError('{0} does not implement mix_and_decompose_1site'.format(type(self).__name__))

    def mix_and_decompose_2site(self, engine, theta, i0, mix_left, mix_right, qtotal_LR=None):
        """``theta -> U, S, VH`` with only the mixed side(s) guaranteed isometric (reference mps_common.py:1754):
        `mixed_svd_2site` if the mixer has it, else built from `mix_and_decompose_1site`."""
        try:
            return self.mixed_svd_2site(engine, theta, i0, mix_left, mix_right, qtotal_LR)
        except NotImplementedError:
            pass
        if not (mix_left or mix_right):
            raise ValueError('Expected mix_left=True and/or mix_right=True.')
        # view the two-site theta as a one-site wave function whose second / first leg is an opaque virtual leg
        as_left = theta.replace_label('(p1.vR)', 'vR')
        as_right = theta.replace_labels(['(vL.p0)', '(p1.vR)'], ['vL', '(p0.vR)'])
        if mix_left and not mix_right:
            U, S, VH, err = self.mix_and_decompose_1site(engine, as_left, i0, move_right=True)
            return U, S, VH.ireplace_label('vR', '(p1.vR)'), err, S
        if mix_right and not mix_left:
            U, S, VH, err = self.mix_and_decompose_1site(engine, as_right, i0 + 1, move_right=False)
            return U.ireplace_label('vL', '(vL.p0)'), S, VH.ireplace_label('(p0.vR)', '(p1.vR)'), err, S
        # both sides: two independent expansions, the bond matrix is what remains of theta between the two isometries
        qtotal_L, qtotal_R = self.determine_qtotal_L_R(theta.qtotal, qtotal_LR)
        U, _, _, err_L = self.mix_and_decompose_1site(engine, as_left, i0, move_right=True)
        _, S_approx, VH, err_R = self.mix_and_decompose_1site(engine, as_right, i0 + 1, move_right=False)
        U = U.gauge_total_charge(1, qtotal_L)
        VH = VH.gauge_total_charge(0, qtotal_R).ireplace_label('(p0.vR)', '(p1.vR)')
        bond = npc.tensordot(U.conj(), theta, axes=['(vL*.p0*)', '(vL.p0)'])
        bond = npc.tensordot(bond, VH.conj(), axes=['(p1.vR)', '(p1*.vR*)'])
        bond.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
        return U, bond / bond.norm(), VH, err_L + err_R, S_approx

    @staticmethod
    def determine_qtotal_L_R(theta_qtotal, qtotal_LR):
        """``qtotal_L + qtotal_R == theta_qtotal`` (reference mps_common.py:1823)."""
        qtotal_L, qtotal_R = (None, None) if qtotal_LR is None else qtotal_LR
        if qtotal_L is None and qtotal_R is None:
            qtotal_L = 0 * theta_qtotal
            qtotal_R = theta_qtotal
        elif qtotal_L is None:
            qtotal_L = theta_qtotal - qtotal_R
        elif qtotal_R is None:
            qtotal_R = theta_qtotal - qtotal_L
        return qtotal_L, qtotal_R


class SubspaceExpansion(Mixer):
    """Direct subspace expansion of a one-site wave function (reference mps_common.py:2082, Hubig et al. 2015): for a
    right move ``theta_expand[(vL.p0), (wR.vR)] = mix_L[wR] LHeff . theta`` is decomposed instead of `theta`; `U`
    spans the expanded space, projecting `VH` back onto ``wR = IdL`` recovers `theta` (up to truncation).  Works on
    one-site wave functions, so single-site DMRG keeps its one-site cost; two-site engines use it through
    :meth:`Mixer.mix_and_decompose_2site`."""
    can_decompose_1site = True

    def mix_and_decompose_1site(self, engine, theta, i0, move_right):
        from ..linalg.truncation import svd_theta
        bond = i0 if move_right else i0 - 1
        mix_L, mix_R, IdL, IdR, explicit_plus_hc = _mix_LR(engine.env.H, bond, np.sqrt(self.amplitude))
        if explicit_plus_hc:
            raise NotImplementedError('explicit_plus_hc MPOs')
        if move_right:
            LHeff = _get_LHeff(engine.env, i0, engine.eff_H).transpose(['(vR*.p0)', 'wR', '(vR.p0*)'])
            if IdL is not None:
                theta_expand = npc.tensordot(LHeff.scale_axis(mix_L, 'wR'), theta, axes=['(vR.p0*)', '(vL.p0)'])
                theta_expand.ireplace_label('(vR*.p0)', '(vL.p0)')
            else:
                wR = LHeff.get_leg('wR')
                stack = [theta.add_trivial_leg(1, 'wR', wR.qconj)]
                proj = np.ones(wR.ind_len, dtype=bool)
                if IdR is not None:
                    proj[IdR] = False
                LHeff = LHeff.copy(deep=True)
                LHeff.iproject(proj, 'wR')
                LHeff = LHeff * np.sqrt(self.amplitude)
                th = npc.tensordot(LHeff, theta, axes=['(vR.p0*)', '(vL.p0)'])
                stack.append(th.ireplace_label('(vR*.p0)', '(vL.p0)'))
                theta_expand = npc.concatenate(stack, axis='wR')
                IdL = 0
            theta_expand = theta_expand.combine_legs(['wR', 'vR'], qconj=-1)
            U, S, VH, err, _ = svd_theta(theta_expand, engine.trunc_params, qtotal_LR=[theta.qtotal, None],
                                         inner_labels=['vR', 'vL'])
            VH = VH.split_legs('(wR.vR)').take_slice(IdL, 'wR')      # back to the original theta
        else:
            RHeff = _get_RHeff(engine.env, i0, engine.eff_H).transpose(['(p1*.vL)', 'wL', '(p1.vL*)'])
            if IdR is not None:
                theta_expand = npc.tensordot(theta, RHeff.scale_axis(mix_R, 'wL'), axes=['(p0.vR)', '(p1*.vL)'])
                theta_expand.ireplace_label('(p1.vL*)', '(p0.vR)')
            else:
                wL = RHeff.get_leg('wL')
                stack = [theta.add_trivial_leg(1, 'wL', wL.qconj)]
                proj = np.ones(wL.ind_len, dtype=bool)
                if IdL is not None:
                    proj[IdL] = False
                RHeff = RHeff.copy(deep=True)
                RHeff.iproject(proj, 'wL')
                RHeff = RHeff * np.sqrt(self.amplitude)
                th = npc.tensordot(theta, RHeff, axes=['(p0.vR)', '(p1*.vL)'])
                stack.append(th.ireplace_label('(p1.vL*)', '(p0.vR)'))
                theta_expand = npc.concatenate(stack, axis='wL')
                IdR = 0
            theta_expand = theta_expand.combine_legs(['vL', 'wL'], qconj=+1)
            U, S, VH, err, _ = svd_theta(theta_expand, engine.trunc_params, qtotal_LR=[None, theta.qtotal],
                                         inner_labels=['vR', 'vL'])
            U = U.split_legs('(vL.wL)').take_slice(IdR, 'wL')
        return U, S, VH, err


class DensityMatrixMixer(Mixer):
    """Mixer perturbing the reduced density matrices with the MPO (reference mps_common.py:1903).

    Options `amplitude` (1e-5), `decay` (2.), `disable_after` (15) as the reference's `Mixer` (:1560)."""
    can_decompose_1site = False   # single-site engines fall back to the two-site theta (reference dmrg.py:1088)

    def mixed_svd_2site(self, engine, theta, i0, mix_left, mix_right, qtotal_LR=[None, None]):
        """Reference mps_common.py:1938."""
        rho_L, rho_R = self.mix_rho(engine, theta, i0, mix_left, mix_right)
        return self.svd_from_rho(engine, rho_L, rho_R, theta, qtotal_LR)

    def mix_rho(self, engine, theta, i0, mix_left, mix_right):
        """Reference mps_common.py:1972."""
        mix_L, mix_R, IdL, IdR, explicit_plus_hc = _mix_LR(engine.env.H, i0, self.amplitude)
        eff_H = engine.eff_H
        if mix_left:
            LHeff = _get_LHeff(engine.env, i0, eff_H)
            rho_L = npc.tensordot(LHeff, theta, axes=['(vR.p0*)', '(vL.p0)'])
            rho_L.ireplace_label('(vR*.p0)', '(vL.p0)')
            rho_c = rho_L.conj()
            rho_L = rho_L.scale_axis(mix_L, 'wR')
            rho_L = npc.tensordot(rho_L, rho_c, axes=[['wR', '(p1.vR)'], ['wR*', '(p1*.vR*)']])
            if IdL is None:
                rho_L = rho_L + npc.tensordot(theta, theta.conj(), axes=['(p1.vR)', '(p1*.vR*)'])
        else:
            rho_L = npc.tensordot(theta, theta.conj(), axes=['(p1.vR)', '(p1*.vR*)'])
        if mix_right:
            RHeff = _get_RHeff(engine.env, i0 + 1, eff_H)
            rho_R = npc.tensordot(theta, RHeff, axes=['(p1.vR)', '(p1*.vL)'])
            rho_R.ireplace_label('(p1.vL*)', '(p1.vR)')
            rho_c = rho_R.conj()
            rho_R = rho_R.scale_axis(mix_R, 'wL')
            rho_R = npc.tensordot(rho_c, rho_R, axes=[['wL*', '(vL*.p0*)'], ['wL', '(vL.p0)']])
            if IdR is None:
                rho_R = rho_R + npc.tensordot(theta.conj(), theta, axes=['(vL*.p0*)', '(vL.p0)'])
        else:
            rho_R = npc.tensordot(theta.conj(), theta, axes=['(vL*.p0*)', '(vL.p0)'])
        return rho_L, rho_R

    def svd_from_rho(self, engine, rho_L, rho_R, theta, qtotal_LR):
        """Reference mps_common.py:2029."""
        chinfo = theta.chinfo
        qtotal_L, qtotal_R = qtotal_LR
        if qtotal_L is None and qtotal_R is None:
            qtotal_R = theta.qtotal
        if qtotal_L is None:
            qtotal_L = chinfo.make_valid(theta.qtotal - qtotal_R)
        elif qtotal_R is None:
            qtotal_R = chinfo.make_valid(theta.qtotal - qtotal_L)
        qtotal_L, qtotal_R = chinfo.make_valid(qtotal_L), chinfo.make_valid(qtotal_R)
        rho_L.itranspose(['(vL.p0)', '(vL*.p0*)'])
        rho_R.itranspose(['(p1.vR)', '(p1*.vR*)'])
        val_L, U = npc.eigh(rho_L)
        U.iset_leg_labels(['(vL.p0)', 'vR'])
        val_L[val_L < 0.] = 0.
        val_L /= np.sum(val_L)
        S_a = np.sqrt(val_L)
        keep_L, _, err_L = truncate(S_a, engine.trunc_params)
        U.iproject(keep_L, axes='vR')
        U = U.gauge_total_charge(1, qtotal_L)
        val_R, Vc = npc.eigh(rho_R)
        Vc.iset_leg_labels(['(p1.vR)', 'vL'])
        VH = Vc.itranspose(['vL', '(p1.vR)'])
        val_R[val_R < 0.] = 0.
        val_R /= np.sum(val_R)
        keep_R, _, err_R = truncate(np.sqrt(val_R), engine.trunc_params)
        VH.iproject(keep_R, axes='vL')
        VH = VH.gauge_total_charge(0, qtotal_R)
        theta = npc.tensordot(U.conj(), theta, axes=['(vL*.p0*)', '(vL.p0)'])
        theta = npc.tensordot(theta, VH.conj(), axes=['(p1.vR)', '(p1*.vR*)'])
        theta.ireplace_labels(['vR*', 'vL*'], ['vL', 'vR'])
        theta /= theta.norm()
        S_a = S_a[keep_L]
        return U, theta, VH, err_L + err_R, S_a
