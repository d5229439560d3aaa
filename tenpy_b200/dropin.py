"""Run the reference's own drivers on the device-resident engine (SURVEY.md section 8b, boundary B1).

The algorithms of tenpy/tenpy reach the tensor engine only through ``from ..linalg import np_conserved as npc``
(tenpy/algorithms/dmrg.py:42, mps_common.py, tebd.py, networks/mps.py, mpo.py, site.py, models/*).  :func:`install` makes
that import resolve to :mod:`tenpy_b200.linalg.np_conserved` / :mod:`tenpy_b200.linalg.charges`, so that the UNMODIFIED
reference files -- ``tenpy.algorithms.dmrg``, ``tebd``, ``mps_common``, ``truncation``, ``krylov_based``, the MPS / MPO /
Site / model classes -- run with every Array in packed HBM and every contraction, SVD, eigh, block move on the CUDA
kernels of ``libb200npc.so``::

    from tenpy_b200 import dropin
    dropin.install()                       # BEFORE the first ``import tenpy``
    import tenpy
    from tenpy.algorithms import dmrg      # the reference's file, now on the B200 engine
    M = tenpy.models.tf_ising.TFIChain({...}); psi = tenpy.networks.mps.MPS.from_product_state(...)
    dmrg.run(psi, M, {...})

How: ``sys.modules['tenpy.linalg.np_conserved']`` and ``['tenpy.linalg.charges']`` are seeded with the engine's modules
(an ``import`` statement consults ``sys.modules`` first, so ``tenpy/linalg/__init__.py:27`` picks them up), and a one-shot
import hook marks ``tenpy.tools.optimization.have_cython_functions = False`` right after that module is executed: the
reference asserts at ``tenpy/linalg/__init__.py:74`` that its ``@use_cython`` decorator ran, which it does not when its own
``np_conserved.py`` is never executed.  Nothing of the reference is modified or copied.

The speed-relevant extension of the engine -- the split-order / identity-environment effective-H matvec -- plugs into the
reference engine through the reference's own hook, the class attribute ``EffectiveH`` (tenpy/algorithms/mps_common.py:
``Sweep.EffectiveH``): :func:`fast_two_site_engine` returns a subclass of the reference's ``TwoSiteDMRGEngine`` whose
``EffectiveH`` inherits the reference's ``TwoSiteH`` and the engine's split-order routes
(:class:`tenpy_b200.algorithms.mps_common.SplitOrderMatvec`, the same code the engine's own ``TwoSiteH`` runs).
"""
import importlib
import importlib.abc
import importlib.util
import os
import sys

__all__ = ['install', 'installed', 'reference_path', 'fast_two_site_engine']

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def reference_path():
    """where the unmodified reference lives: ``$TENPY_REFERENCE`` (a checkout or install of tenpy/tenpy), the copy
    ``build()`` placed under ``oracle/_ref`` or the offline install ``baseline/_ref``; None if none is there"""
    cands = [os.environ.get('TENPY_REFERENCE'), os.path.join(_ROOT, 'oracle', '_ref'), os.path.join(_ROOT, 'baseline', '_ref')]
    for c in cands:
        if c and os.path.isdir(os.path.join(c, 'tenpy')):
            return c
    return None


class _MarkNoCython(importlib.abc.MetaPathFinder):
    """one-shot post-import hook on ``tenpy.tools.optimization`` (see the module doc string)"""

    name = 'tenpy.tools.optimization'

    def find_spec(self, fullname, path, target=None):
        if fullname != self.name:
            return None
        sys.meta_path.remove(self)
        spec = importlib.util.find_spec(fullname)
        if spec is None:
            return None
        inner = spec.loader

        class _Loader(importlib.abc.Loader):
            def create_module(self, sp):
                return inner.create_module(sp)

            def exec_module(self, module):
                inner.exec_module(module)
                module.have_cython_functions = False      # the engine's modules carry no @use_cython hooks

        spec.loader = _Loader()
        return spec


def installed():
    npc = sys.modules.get('tenpy.linalg.np_conserved')
    return npc is not None and getattr(npc, '__name__', '') == 'tenpy_b200.linalg.np_conserved'


def install(path=None):
    """Seed the engine's modules under the reference's names; must run before the first ``import tenpy``.  `path`: the
    reference checkout / install to put on ``sys.path`` (default :func:`reference_path`).  Returns the path used."""
    if installed():
        return path or reference_path()
    if 'tenpy' in sys.modules:
        raise RuntimeError('tenpy_b200.dropin.install() has to run before the first `import tenpy`')
    from .linalg import np_conserved, charges
    sys.modules['tenpy.linalg.np_conserved'] = np_conserved
    sys.modules['tenpy.linalg.charges'] = charges
    sys.meta_path.insert(0, _MarkNoCython())
    path = path or reference_path()
    if path is not None and path not in sys.path:
        sys.path.insert(0, path)
    return path


def fast_two_site_engine():
    """The reference's ``TwoSiteDMRGEngine`` with the device-optimised effective Hamiltonian plugged in at the reference's
    own extension point ``EffectiveH``.  Call after :func:`install`."""
    if not installed():
        raise RuntimeError('call tenpy_b200.dropin.install() first')
    import numpy as np
    from tenpy.algorithms import dmrg as ref_dmrg
    from tenpy.algorithms import mps_common as ref_common
    from .algorithms.mps_common import SplitOrderMatvec

    class B200TwoSiteH(SplitOrderMatvec, ref_common.TwoSiteH):
        """reference ``TwoSiteH`` (same constructor, attributes, `combine_theta`, `update_LP` ...); `matvec` applies
        ``LP``, ``W0 W1``, ``RP`` to the split theta without the identity components of the environments where that is
        cheaper (`SplitOrderMatvec`), the reference order otherwise."""

        def __init__(self, env, i0, combine=False, move_right=True):
            super().__init__(env, i0, combine, move_right)
            self._H_mpo = env.H

        def matvec(self, theta):
            # the split-order routes are real-only: a complex theta or MPO takes the reference's order
            if self.combine and np.dtype(self.dtype).kind != 'c' and np.dtype(theta.dtype).kind != 'c' and \
                    self._use_split(theta):
                return self._matvec_split(theta, theta.get_leg_labels())
            return super().matvec(theta)

    class B200TwoSiteDMRGEngine(ref_dmrg.TwoSiteDMRGEngine):
        EffectiveH = B200TwoSiteH

    return B200TwoSiteDMRGEngine
