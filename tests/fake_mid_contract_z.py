"""TEST DOUBLE of ``b200_mid_contract2_z`` -- test infrastructure, never shipped, never imported by the package.

A numpy einsum with the argument list of :meth:`tenpy_b200._lib.DeviceLib.mid_contract2_z`, added by :func:`install` to
an instance of the test double of the device library (tests/fake_device.py), so that the host logic of the complex
split-order matvec runs in the ``-m "not gpu"`` suite.  The GPU tests run the CUDA kernel.
"""
import types

import numpy as np


def mid_contract2_z(self, K1, K2, N1, N2, C1, outer, inner, M, T1, T2, OUT1, OUT2):
    """[OUT1; OUT2][o, n, i] = sum_k M[n, k] [T1; T2][o, k, i] on planar complex M, T1, T2; OUT2 planar, OUT1 the real
    embedding [[Yr, -Yi], [Yi, Yr]] of Y[(o, n // C1), (n % C1, i)] (include/b200npc.h)"""
    self._count('mid_contract2_z')
    N, K = N1 + N2, K1 + K2
    m = M.numpy()[:2 * N * K]
    m = m[:N * K].reshape(N, K) + 1.j * m[N * K:].reshape(N, K)
    parts = []
    for Kx, T in ((K1, T1), (K2, T2)):
        if Kx:
            n = outer * Kx * inner
            t = T.numpy()[:2 * n]
            parts.append((t[:n] + 1.j * t[n:]).reshape(outer, Kx, inner))
    res = np.einsum('nk,oki->oni', m, np.concatenate(parts, axis=1))
    if N1:
        Y = res[:, :N1].reshape(outer * (N1 // C1), C1 * inner)
        emb = np.block([[Y.real, -Y.imag], [Y.imag, Y.real]])
        OUT1.numpy()[:emb.size] = emb.reshape(-1)
    if N2:
        y = res[:, N1:].reshape(-1)
        OUT2.numpy()[:2 * y.size] = np.concatenate([y.real, y.imag])


def install(lib):
    """give the test double `lib` the method ``mid_contract2_z``; returns `lib`"""
    lib.mid_contract2_z = types.MethodType(mid_contract2_z, lib)
    return lib
