"""tenpy_b200 -- an H100-native (sm_90a) block-sparse tensor engine for the two-site DMRG hot path.

Mirrors the reference interface of tenpy/tenpy for that path (``linalg.np_conserved``, ``linalg.charges``,
``linalg.krylov_based``, ``linalg.truncation``, ``algorithms.mps_common.TwoSiteH``, ``algorithms.dmrg``,
``networks.mpo.MPOEnvironment``); all floating point work runs in the CUDA library ``csrc/libb200npc.so``
behind the C ABI of ``include/b200npc.h``.  There is no CPU fallback.
"""
__version__ = '0.1.0'
