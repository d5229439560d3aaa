"""TEST DOUBLE of the complex Hermitian block eigh of the device library -- test infrastructure, never shipped.

`FakeEighZDeviceLib` is the complex test double of tests/fake_device_complex.py plus a numpy ``block_eigh_z`` (planar
real / imaginary buffers in and out).  Like the kernel, it diagonalises (A + A^H) / 2 and returns W ascending and the
eigenvectors in the columns of V.  Installed by the complex eigh / DMRG tests and by tests/dropin/run_dmrg_complex.py in
``fake`` mode.
"""
import numpy as np
import torch

from fake_device_complex import FakeComplexDeviceLib


class FakeEighZDeviceLib(FakeComplexDeviceLib):
    name = 'FAKE numpy test double with complex decompositions and complex eigh (tests only)'

    def block_eigh_z(self, n, a_off, w_off, v_off, A_re, A_im, W, V_re, V_im):
        self._count('block_eigh_z')
        ar, ai, w, vr, vi = A_re.numpy(), A_im.numpy(), W.numpy(), V_re.numpy(), V_im.numpy()
        for i in range(len(n)):
            ni = int(n[i])
            sl = slice(a_off[i], a_off[i] + ni * ni)
            blk = (ar[sl] + 1.j * ai[sl]).reshape(ni, ni)
            ww, vv = np.linalg.eigh(0.5 * (blk + blk.conj().T))
            w[w_off[i]:w_off[i] + ni] = ww
            vr[v_off[i]:v_off[i] + ni * ni] = vv.real.reshape(-1)
            vi[v_off[i]:v_off[i] + ni * ni] = vv.imag.reshape(-1)
        return np.ones(len(n), dtype=np.int32)


def install():
    """select the double as the device library; returns (lib, restore) -- `restore()` puts the previous state back.
    Uninitialised buffers are poisoned with NaN, like the ``fake_device`` fixture of tests/conftest.py does."""
    from tenpy_b200 import backend
    old_lib, old_empty = backend._state['lib'], backend.empty
    lib = backend.use_library(FakeEighZDeviceLib())
    backend.empty = lambda n: torch.full((int(n),), float('nan'), dtype=torch.float64)

    def restore():
        backend.empty = old_empty
        backend.use_library(old_lib)
    return lib, restore
