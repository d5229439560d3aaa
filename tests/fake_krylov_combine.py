"""TEST DOUBLE of ``b200_krylov_combine_f64`` -- test infrastructure, never shipped, never imported by the package.

numpy with the argument list of :meth:`tenpy_b200._lib.DeviceLib.krylov_combine`, added by :func:`install` to an instance
of the test double of the device library (tests/fake_device.py), so that the Lanczos time evolution and the TDVP engines
run in the ``-m "not gpu"`` suite.  The test double keeps its buffers in host memory, so the addresses of the pointer
table are read directly.  The argument checks are those of the kernel.  The GPU tests run the CUDA kernel.
"""
import ctypes
import types

import numpy as np

from tenpy_b200 import _lib


def _view(addr, count):
    return np.ctypeslib.as_array((ctypes.c_double * count).from_address(int(addr)))


def krylov_combine(self, n, in_planes, ptr_host, ptr_dev, coef_dev, OUT):
    """OUT[:2n] = sum_k c_k v_k, c_k = coef_dev[2k] + i coef_dev[2k+1] (include/b200npc.h)"""
    ptrs = [int(p) for p in np.asarray(ptr_host, dtype=np.int64)]
    nvec = len(ptrs)
    if not 1 <= nvec <= 64 or in_planes not in (1, 2) or n < 0:
        raise _lib.B200Error('libb200npc error 1: krylov_combine: bad arguments')
    if n == 0:
        return
    o0 = OUT.data_ptr()
    for p in ptrs:
        if p == 0 or (p < o0 + 16 * n and o0 < p + 8 * in_planes * n):
            raise _lib.B200Error('libb200npc error 1: krylov_combine: out overlaps a vector')
    self._count('krylov_combine')
    c = coef_dev.numpy()[:2 * nvec]
    acc = np.zeros(n, dtype=np.complex128)
    for k, p in enumerate(ptrs):
        v = _view(p, in_planes * n)
        x = v if in_planes == 1 else v[:n] + 1.j * v[n:]
        acc += complex(c[2 * k], c[2 * k + 1]) * x
    out = OUT.numpy()
    out[:n] = acc.real
    out[n:2 * n] = acc.imag


def install(lib):
    """give the test double `lib` the method ``krylov_combine``; returns `lib`"""
    lib.krylov_combine = types.MethodType(krylov_combine, lib)
    return lib
