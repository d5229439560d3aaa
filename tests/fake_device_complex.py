"""TEST DOUBLE of the complex decompositions of the device library -- test infrastructure, never shipped.

`FakeComplexDeviceLib` is the numpy test double of tests/fake_device.py plus numpy versions of ``block_svd_z`` and
``block_qr_z`` (planar real / imaginary buffers in and out).  The SVD emulates the kernel's deflation contract including
its orientation: a block with m >= n is orthogonalised on its columns (``transposed`` = 1, the vectors of the negligible
directions are left as ZERO columns of U), other blocks on their rows (zero rows of VT), so both completion paths of
``npc.svd`` run on the CPU.  Installed by the ``fake_device_z`` fixture of the complex tests and by
tests/dropin/run_tebd_real.py in ``fake`` mode.
"""
import numpy as np
import torch

from fake_device import FakeDeviceLib


class FakeComplexDeviceLib(FakeDeviceLib):
    name = 'FAKE numpy test double with complex decompositions (tests only)'

    def block_svd_z(self, m, n, a_off, u_off, s_off, vt_off, A_re, A_im, U_re, U_im, S, VT_re, VT_im):
        self._count('block_svd_z')
        ar, ai, s = A_re.numpy(), A_im.numpy(), S.numpy()
        ur, ui, vr, vi = U_re.numpy(), U_im.numpy(), VT_re.numpy(), VT_im.numpy()
        nact = np.zeros(len(m), dtype=np.int32)
        transp = np.zeros(len(m), dtype=np.int32)
        for i in range(len(m)):
            mi, ni = int(m[i]), int(n[i])
            k = min(mi, ni)
            sl = slice(a_off[i], a_off[i] + mi * ni)
            blk = (ar[sl] + 1.j * ai[sl]).reshape(mi, ni)
            uu, ss, vv = np.linalg.svd(blk, full_matrices=False)
            defl = max(16 * 2.220446049250313e-16 * np.sqrt(max(mi, ni)), self.deflation_tol) * np.linalg.norm(blk) \
                if self.deflation else -1.
            r = int(np.sum(ss > defl))
            uu, vv = uu.copy(), vv.copy()
            if mi >= ni:
                transp[i] = 1
                uu[:, r:] = 0.
            else:
                vv[r:] = 0.
            nact[i] = r
            ur[u_off[i]:u_off[i] + mi * k] = uu.real.reshape(-1)
            ui[u_off[i]:u_off[i] + mi * k] = uu.imag.reshape(-1)
            s[s_off[i]:s_off[i] + k] = ss
            vr[vt_off[i]:vt_off[i] + k * ni] = vv.real.reshape(-1)
            vi[vt_off[i]:vt_off[i] + k * ni] = vv.imag.reshape(-1)
        return np.ones(len(m), dtype=np.int32), nact, transp

    def block_qr_z(self, m, n, a_off, q_off, r_off, A_re, A_im, Q_re, Q_im, R_re, R_im):
        """numpy complex QR on planar buffers, R with a real non-negative diagonal"""
        self._count('block_qr_z')
        ar, ai = A_re.numpy(), A_im.numpy()
        for i in range(len(m)):
            mi, ni = int(m[i]), int(n[i])
            k = min(mi, ni)
            sl = slice(a_off[i], a_off[i] + mi * ni)
            qq, rr = np.linalg.qr((ar[sl] + 1.j * ai[sl]).reshape(mi, ni))
            d = np.diag(rr)
            ad = np.abs(d)
            ph = np.where(ad > 0., d / np.where(ad > 0., ad, 1.), 1.)
            qq = qq * ph[None, :]
            rr = rr * ph.conj()[:, None]
            for buf, part in ((Q_re, qq.real), (Q_im, qq.imag)):
                buf.numpy()[q_off[i]:q_off[i] + mi * k] = part.reshape(-1)
            for buf, part in ((R_re, rr.real), (R_im, rr.imag)):
                buf.numpy()[r_off[i]:r_off[i] + k * ni] = part.reshape(-1)


def install():
    """select the double as the device library; returns (lib, restore) -- `restore()` puts the previous state back.
    Uninitialised buffers are poisoned with NaN, like the ``fake_device`` fixture of tests/conftest.py does."""
    from tenpy_b200 import backend
    old_lib, old_empty = backend._state['lib'], backend.empty
    lib = backend.use_library(FakeComplexDeviceLib())
    backend.empty = lambda n: torch.full((int(n),), float('nan'), dtype=torch.float64)

    def restore():
        backend.empty = old_empty
        backend.use_library(old_lib)
    return lib, restore
