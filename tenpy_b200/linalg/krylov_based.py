"""Lanczos ground state search and time evolution on device-resident Arrays.

Host-side mirror of the reference ``tenpy/linalg/krylov_based.py`` (class `LanczosGroundState` :584,
`LanczosEvolution` :718, `KrylovBased` :30): same options (`N_min`, `N_max`, `P_tol`, `E_tol`, `min_gap`, `N_cache`, `reortho`,
`cutoff`, `E_shift`), same three-term recurrence, same convergence test (`_converged` :677) and same
result assembly (`_calc_result_full` :160).  The control flow and the tridiagonal ``eigh`` (at most
``(N_max+1)^2`` numbers) stay on the host, as in the reference; every vector operation is a kernel over the
packed HBM buffers (``matvec`` = 2 grouped GEMMs, `inner` / `norm` = dot kernels, axpy / scal).
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import logging

import numpy as np

from . import np_conserved as npc
from .. import backend

logger = logging.getLogger(__name__)

__all__ = ['KrylovBased', 'LanczosGroundState', 'LanczosEvolution', 'lanczos']

DEVICE_SCALARS_DEFAULT = True    # Lanczos option `device_scalars`: (alpha, beta) stay on the device, read back in chunks


def _pack(v, lay=None):
    """A complex Krylov vector on the device-scalar route: the ComplexArray `v` with both parts in ONE device buffer
    ``[re | im]`` of ``2 lay.size`` elements on the block table `lay` (default: the union of the tables of its parts).
    For a Hermitian operator every step of the recurrence is a real operation on that buffer: ``alpha = Re<v|Hv>`` is the
    real dot product of the packed planes, and the update, the normalisation and the result assembly have real
    coefficients.  Returns the ComplexArray whose parts are views of the two halves, with the buffer as ``_kbuf``, or
    ``None`` if the table of `v` differs from `lay`."""
    union, (re, im) = npc._planes(v)
    if lay is None:
        lay = union
    elif not (union is lay or union.same_blocks(lay)):
        return None
    n = lay.size
    buf = backend.empty(2 * n)
    buf[:n].copy_(re)
    buf[n:].copy_(im)
    out = npc._from_planes(v.legs, v.qtotal, lay, (buf[:n], buf[n:]), v.get_leg_labels())
    out._kbuf = buf
    return out


def _flat(v):
    """``(n, buffer)``: the real Array `v`, or the packed ComplexArray (:func:`_pack`), as one real device vector"""
    kbuf = getattr(v, '_kbuf', None)
    if kbuf is not None:
        return kbuf.numel(), kbuf
    return v._layout.size, v._buf


class KrylovBased:
    """Base class: option parsing, cache and result assembly (reference krylov_based.py:30)."""

    def __init__(self, H, psi0, options):
        self.H = H
        self.psi0 = psi0.copy()
        self._psi0_norm = None
        self.options = options = dict(options) if options is not None else {}
        self.N_min = int(options.get('N_min', 2))
        self.N_max = int(options.get('N_max', 20))
        self.N_cache = self.N_max
        self.P_tol = float(options.get('P_tol', 1.e-14))
        self.min_gap = float(options.get('min_gap', 1.e-12))
        self.reortho = bool(options.get('reortho', False))
        self.E_shift = options.get('E_shift', None)
        if self.E_shift is not None:
            raise NotImplementedError('E_shift')
        if self.N_min < 2:
            raise ValueError('Should perform at least 2 steps.')
        self._cutoff = float(options.get('cutoff', np.finfo(np.float64).eps * 100))
        self._cache = []
        self.Es = np.zeros([self.N_max, self.N_max], dtype=np.float64)
        self._h_krylov = np.zeros([self.N_max + 1, self.N_max + 1], dtype=np.float64)
        self._result_krylov = None

    def _to_cache(self, psi):
        cache = self._cache
        cache.append(psi)
        if len(cache) > self.N_cache:
            cache.pop(0)

    def _calc_result_full(self, N):
        """``psi_f = sum_k result_krylov[k] psi[k]`` (reference krylov_based.py:160)."""
        vf = self._result_krylov
        assert N == len(vf) > 1
        psif = self.psi0 * vf[0]
        if np.dtype(psif.dtype).kind != 'c' and any(np.dtype(c.dtype).kind == 'c' for c in self._cache):
            psif = psif.astype(np.complex128)        # a real start vector, a complex operator
        len_cache = len(self._cache)
        for k in range(1, min(len_cache + 1, N)):
            psif.iadd_prefactor_other(vf[N - k], self._cache[-k])
        self._cache = []
        self._rebuild_krylov_for_result_full(psif, N - len_cache - 1)
        if getattr(self, 'device_scalars', False) and np.dtype(psif.dtype).kind == 'c':
            psif = _pack(psif)
        if getattr(self, 'device_scalars', False) and _flat(psif)[0]:
            # normalisation without a host round trip (same arithmetic: |psi|^2 by the dot kernel, x *= 1 / sqrt(.)); the
            # conditioning warning of the reference is raised when somebody reads `norm_check()` (the DMRG engine: at the
            # end of the sweep)
            lib = backend.get_lib()
            n2 = backend.empty(1)
            size, buf = _flat(psif)
            lib.dot(size, buf, buf, backend.dot_scratch(), n2)
            lib.scal_rsqrt_dev(size, n2, buf)
            self._result_norm2_dev = n2
            return psif
        psif_norm = npc.norm(psif)
        if abs(1. - psif_norm) > 1.e-5:
            logger.warning('poorly conditioned H matrix in KrylovBased! |psi_0| = %f', psif_norm)
        psif.iscale_prefactor(1. / psif_norm)
        return psif

    def norm_check(self):
        """the deferred conditioning test of :meth:`_calc_result_full` (synchronises); returns the norm or ``None``"""
        n2 = getattr(self, '_result_norm2_dev', None)
        if n2 is None:
            return None
        self._result_norm2_dev = None
        psif_norm = float(np.sqrt(backend.read_scalar(n2)))
        if abs(1. - psif_norm) > 1.e-5:
            logger.warning('poorly conditioned H matrix in KrylovBased! |psi_0| = %f', psif_norm)
        return psif_norm


class LanczosGroundState(KrylovBased):
    """Lanczos algorithm for the ground state of a hermitian `H` (reference krylov_based.py:584).

    `H` needs a method ``matvec(Array) -> Array``; `psi0` is the start vector."""

    def __init__(self, H, psi0, options):
        super().__init__(H, psi0, options)
        self.E_tol = float(self.options.get('E_tol', np.inf))
        self.N_cache = int(self.options.get('N_cache', self.N_max))
        if self.N_cache < 2:
            raise ValueError('Need to cache at least two vectors.')
        # extension (opt-in): keep (alpha, beta) on the device and read them back in chunks, see _build_krylov_device
        self.device_scalars = bool(self.options.get('device_scalars', DEVICE_SCALARS_DEFAULT))
        self.sync_every = max(1, int(self.options.get('sync_every', 2)))

    def run(self):
        """Returns ``(E0, psi0, N)`` (reference krylov_based.py:614)."""
        N = self._build_krylov()
        E0 = self.Es[N - 1, 0]
        if N == 1:
            return E0, self.psi0.copy(), N
        return E0, self._calc_result_full(N), N

    def _build_krylov_device(self):
        """The recurrence of :meth:`_build_krylov` without a host round trip per iteration: ``alpha_k`` (written by the
        dot kernel) and ``|w|^2`` stay in a small device array, the update and the normalisation read them there
        (``b200_lanczos_update_dev_f64``, ``b200_scal_rsqrt_dev_f64``; bit-identical arithmetic).  The scalars come
        back in chunks -- after the first `N_min` iterations (nothing can converge earlier), then every `sync_every`
        -- and the reference's bookkeeping (tridiagonal `eigh`, `_converged`, breakdown test) is replayed on the host
        for every ``k`` of the chunk in order: the run stops at exactly the ``k`` the reference stops at, iterations
        enqueued beyond it are discarded (their vectors are dropped from the cache).  Returns ``N`` or ``None`` if the
        vectors do not share one block layout (caller falls back to the host-scalar loop)."""
        h = self._h_krylov
        lib = backend.get_lib()
        cplx = np.dtype(self.psi0.dtype).kind == 'c'
        if cplx:
            self.psi0 = _pack(self.psi0)          # normalised in place below, like a real start vector
        w = self.psi0
        lay = w.re._layout if cplx else w._layout
        if lay.nblocks == 0:
            raise ValueError('Norm of self.psi0 too small: 0.0')
        size = _flat(w)[0]
        # sc[2k] = alpha_k, sc[2k+1] = |w_k|^2 = beta_{k+1}^2; last entry: |psi0|^2 -- the start vector is normalised on the
        # device as well (same arithmetic as `npc.norm` + `iscale_prefactor`), its norm is tested with the first chunk of
        # scalars: no host round trip before the first `N_min` matvecs are enqueued
        sc = backend.zeros(2 * self.N_max + 1)
        nrm2_0 = sc[2 * self.N_max:2 * self.N_max + 1]
        scratch = backend.dot_scratch()
        lib.dot(size, _flat(w)[1], _flat(w)[1], scratch, nrm2_0)
        done_k = 0                                     # iterations whose scalars have been processed on the host
        k = 0
        while k < self.N_max:
            stop_at = self.N_min if k < self.N_min else min(self.N_max, k + self.sync_every)
            while k < stop_at:
                lib.scal_rsqrt_dev(size, nrm2_0 if k == 0 else sc[2 * k - 1:2 * k], _flat(w)[1])
                self._to_cache(w)
                w = self.H.matvec(w)
                v1 = self._cache[-1]
                if cplx:
                    w = _pack(w if np.dtype(w.dtype).kind == 'c' else w.astype(np.complex128), lay)
                elif np.dtype(w.dtype).kind == 'c' or not (w._layout is v1._layout or
                                                           w._layout.same_blocks(v1._layout)):
                    w = None                                  # (a real start vector, a complex operator: host loop)
                if w is None:
                    if self._psi0_norm is None:
                        self._psi0_norm = float(np.sqrt(backend.read_scalar(nrm2_0)))
                    return None
                lib.dot(size, _flat(w)[1], _flat(v1)[1], scratch, sc[2 * k:2 * k + 1])
                v0 = _flat(self._cache[-2])[1] if k > 0 else None
                lib.lanczos_update_dev(size, sc[2 * k:2 * k + 1], _flat(v1)[1],
                                       sc[2 * k - 1:2 * k] if k > 0 else None, v0, _flat(w)[1], scratch,
                                       sc[2 * k + 1:2 * k + 2])
                k += 1
            vals = backend.to_host(sc)                                # the one synchronisation of this chunk
            if done_k == 0:
                beta0 = float(np.sqrt(vals[-1]))
                if not beta0 >= self._cutoff:
                    raise ValueError('Norm of self.psi0 too small: {0!s}'.format(beta0))
                if self._psi0_norm is None:
                    self._psi0_norm = beta0
            check = getattr(self.H, 'deferred_check', None)
            if check is not None:
                check()                                               # tests the operator postponed to this point
            for kk in range(done_k, k):
                h[kk, kk] = vals[2 * kk]
                # the tridiagonal eigen-problem of step kk is needed for the convergence test of steps kk and kk + 1 (which
                # can only trigger from step N_min - 1 on) and for the result: skipped for the first N_min - 2 steps
                solved = kk + 2 >= self.N_min
                if solved:
                    self._calc_result_krylov(kk)
                beta = float(np.sqrt(vals[2 * kk + 1]))
                h[kk, kk + 1] = h[kk + 1, kk] = beta
                if not np.isfinite(beta) or abs(beta) < self._cutoff or (kk + 1 >= self.N_min and self._converged(kk)):
                    if not solved:
                        self._calc_result_krylov(kk)
                    for _ in range(k - (kk + 1)):                     # vectors of the discarded iterations
                        self._cache.pop()
                    return kk + 1
            done_k = k
        return k

    def _build_krylov(self):
        """Reference krylov_based.py:645."""
        if self.device_scalars and not self.reortho and self.N_cache >= self.N_max:
            N = self._build_krylov_device()
            if N is not None:
                return N
            self._cache = []
        h = self._h_krylov
        w = self.psi0
        beta = npc.norm(w)
        if beta < self._cutoff:
            raise ValueError('Norm of self.psi0 too small: {0!s}'.format(beta))
        if self._psi0_norm is None:
            self._psi0_norm = beta
        k = 0
        for k in range(self.N_max):
            w.iscale_prefactor(1. / beta)
            self._to_cache(w)
            w = self.H.matvec(w)
            # (Re: a ComplexArray gives a complex inner product, real up to rounding for a Hermitian H)
            alpha = float(np.real(npc.inner(w, self._cache[-1], axes='range', do_conj=True)))
            if k == 0 and getattr(self.H, 'deferred_check', None) is not None:
                self.H.deferred_check()                                # tests the operator postponed to its first read-back
            h[k, k] = alpha
            self._calc_result_krylov(k)
            fused = (not self.reortho) and np.dtype(w.dtype).kind != 'c' and \
                w._layout.same_blocks(self._cache[-1]._layout) and \
                (k == 0 or w._layout.same_blocks(self._cache[-2]._layout))
            if fused:
                # w -= alpha v_k + beta v_{k-1};  beta' = |w|   in ONE pass (b200_lanczos_update_f64)
                lib = backend.get_lib()
                out = backend.scalar_out()
                v0 = self._cache[-2]._buf if k > 0 else None
                lib.lanczos_update(w._layout.size, alpha, self._cache[-1]._buf, beta if k > 0 else 0., v0, w._buf,
                                   backend.dot_scratch(), out)
                beta = float(np.sqrt(backend.read_scalar(out)))
            else:
                w.iadd_prefactor_other(-alpha, self._cache[-1])
                if self.reortho:
                    for c in self._cache[:-1]:
                        w.iadd_prefactor_other(-npc.inner(c, w, axes='range', do_conj=True), c)
                elif k > 0:
                    w.iadd_prefactor_other(-beta, self._cache[-2])
                beta = npc.norm(w)
            h[k, k + 1] = h[k + 1, k] = beta
            if abs(beta) < self._cutoff or (k + 1 >= self.N_min and self._converged(k)):
                break
        return k + 1

    def _converged(self, k):
        """Reference krylov_based.py:677."""
        v0 = self._result_krylov
        E = self.Es[k, :]
        RitzRes = abs(v0[k]) * self._h_krylov[k, k + 1]
        gap = max(E[1] - E[0], self.min_gap)
        P_err = (RitzRes / gap)**2
        Delta_E0 = self.Es[k - 1, 0] - E[0]
        return P_err < self.P_tol and Delta_E0 < self.E_tol

    def _rebuild_krylov_for_result_full(self, psif, N_max):
        """Reference krylov_based.py:686 (only needed if N_cache < N)."""
        vf = self._result_krylov
        h = self._h_krylov
        w = self.psi0
        beta = 0.
        for k in range(0, N_max):
            self._to_cache(w)
            w = self.H.matvec(w)
            alpha = h[k, k]
            w.iadd_prefactor_other(-alpha, self._cache[-1])
            if self.reortho:
                for c in self._cache[:-1]:
                    w.iadd_prefactor_other(-npc.inner(c, w, axes='range', do_conj=True), c)
            elif k > 0:
                w.iadd_prefactor_other(-beta, self._cache[-2])
            beta = h[k, k + 1]
            w.iscale_prefactor(1. / beta)
            psif.iadd_prefactor_other(vf[k + 1], w)

    def _calc_result_krylov(self, k):
        """Ground state of the tridiagonal ``h[:k+1, :k+1]`` on the host (reference krylov_based.py:705)."""
        h = self._h_krylov
        if k == 0:
            self.Es[0, 0] = h[0, 0]
            self._result_krylov = np.ones(1, np.float64)
        else:
            E_kr, v_kr = np.linalg.eigh(h[:k + 1, :k + 1])
            self.Es[k, :k + 1] = E_kr
            self._result_krylov = v_kr[:, 0]


class LanczosEvolution(LanczosGroundState):
    """``expm(delta H) psi0`` for a hermitian `H` by Lanczos (reference krylov_based.py:718).

    The recurrence is the one of :class:`LanczosGroundState` (on the device-scalar route :meth:`_build_krylov_device`,
    which replays :meth:`_calc_result_krylov` / :meth:`_converged` below on the host and stops at the ``k`` the reference
    stops at); ``_h_krylov`` stays real.  In the Krylov basis the result is ``expm(delta h) e_0``, converged when its
    last component is below `P_tol`.  On the device-scalar route the result ``sum_k c_k v_k`` with complex ``c_k`` is
    assembled from the cached vectors by ONE kernel (``b200_krylov_combine_f64``; a real start vector gives a complex
    result) and normalised on the device; the conditioning test is deferred to :meth:`norm_check` as for the ground
    state.  Otherwise (vectors on different block tables, ``N_cache < N_max``, `reortho`) the host-scalar assembly of
    :meth:`KrylovBased._calc_result_full` runs.  Options as for :class:`LanczosGroundState`; `E_tol` and `min_gap` are
    ignored."""

    def __init__(self, H, psi0, options):
        super().__init__(H, psi0, options)
        self._result_norm = 1.
        self.delta = None            # set in run()
        self._on_device = False      # the last recurrence ran on the device-scalar route

    def run(self, delta, normalize=None):
        """Returns ``(psi_f, N)``: ``psi_f`` approximates ``expm(delta H) psi0``, normalised if `normalize` (default:
        ``Re(delta) == 0``), else with the norm ``|psi0| |expm(delta h) e_0|`` (reference krylov_based.py:757)."""
        self.delta = delta
        N = self._build_krylov()
        if N == 1:
            result_full = self._result_krylov[0] * self.psi0            # _result_krylov[0] is only a phase
        else:
            result_full = self._calc_result_full(N)
        if normalize is None:
            normalize = np.real(delta) == 0.
        if normalize:
            return result_full, N
        scale = float(self._psi0_norm * self._result_norm)
        kbuf = getattr(result_full, '_kbuf', None)
        if kbuf is not None:
            backend.get_lib().scal(kbuf.numel(), scale, kbuf)
            return result_full, N
        return scale * result_full, N

    def _build_krylov_device(self):
        N = super()._build_krylov_device()
        self._on_device = N is not None
        return N

    def _calc_result_full(self, N):
        """``psi_f = sum_k result_krylov[k] psi[k]`` (reference krylov_based.py:160) in one kernel on the device-scalar
        route: the terms in the reference's order (``psi[0]``, then the cache from its end), the result packed
        ``[re | im]`` (:func:`_pack`) and normalised without a host round trip."""
        cache = self._cache
        if not self._on_device or len(cache) != N:
            return super()._calc_result_full(N)
        order = [0] + list(range(N - 1, 0, -1))
        v0 = cache[0]
        packed = getattr(v0, '_kbuf', None) is not None
        lay = v0.re._layout if packed else v0._layout
        n = lay.size
        vf = np.asarray(self._result_krylov, dtype=np.complex128)[order]
        coef = np.empty(2 * N, dtype=np.float64)
        coef[0::2], coef[1::2] = vf.real, vf.imag
        ptrs = np.array([_flat(cache[k])[1].data_ptr() for k in order], dtype=np.int64)
        lib = backend.get_lib()
        out = backend.empty(2 * n)
        lib.krylov_combine(n, 2 if packed else 1, ptrs, backend.to_device(ptrs), backend.to_device(coef), out)
        self._cache = []
        psif = npc._from_planes(v0.legs, v0.qtotal, lay, (out[:n], out[n:]), v0.get_leg_labels())
        psif._kbuf = out
        n2 = backend.empty(1)
        lib.dot(2 * n, out, out, backend.dot_scratch(), n2)
        lib.scal_rsqrt_dev(2 * n, n2, out)
        self._result_norm2_dev = n2
        return psif

    def _calc_result_krylov(self, k):
        """``expm(delta h) e_0`` for ``h = _h_krylov[:k+1, :k+1]``, normalised (reference krylov_based.py:797)."""
        h = self._h_krylov
        delta = self.delta
        if k == 0:
            exp_dE = np.exp(delta * h[0, 0])
            self._result_norm = np.abs(exp_dE)
            self._result_krylov = np.array([exp_dE / self._result_norm])
        else:
            E_kr, v_kr = np.linalg.eigh(h[:k + 1, :k + 1])
            exp_dH_e0 = np.dot(v_kr, np.exp(E_kr * delta) * np.conj(v_kr[0, :]))
            self._result_norm = np.linalg.norm(exp_dH_e0)
            self._result_krylov = exp_dH_e0 / self._result_norm

    def _converged(self, k):
        """Reference krylov_based.py:821."""
        return np.abs(self._result_krylov[k]) < self.P_tol


def lanczos(H, psi, options={}):
    """Function wrapper (reference krylov_based.py `lanczos`)."""
    return LanczosGroundState(H, psi, options).run()
