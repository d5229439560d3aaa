"""TEST DOUBLE of the device library -- test infrastructure, never shipped, never imported by the package.

`FakeDeviceLib` has the method surface of :class:`tenpy_b200._lib.DeviceLib` but executes every call
with numpy on CPU ``torch`` tensors.  It exists so that the HOST logic of tenpy_b200 (charge bookkeeping,
block layouts, index plans, the DMRG driver) can be unit-tested in the ``-m "not gpu"`` suite on a box
without a GPU.  It is installed by the ``fake_device`` fixture of ``tests/conftest.py`` through
``backend.use_library``; the product never selects it by itself, and no GPU test uses it: the parity
tests proper (``-m gpu``) run the real CUDA kernels and compare against ``oracle/``.

The contraction *plan* (integer bookkeeping) is still built by the real host code of
``libb200npc.so`` (``b200_tdot_plan_create`` needs no device), so that code is covered here too.
"""
import ctypes

import numpy as np
import torch

from tenpy_b200 import _lib


class _FakePlan:
    def __init__(self, real):
        self.real = real
        self.n_c, self.n_pairs, self.c_size, self.flops = real.n_c, real.n_pairs, real.c_size, real.flops
        self.c_qdata, self.c_off, self.c_rows, self.c_cols = real.c_qdata, real.c_off, real.c_rows, real.c_cols
        self._pairs = real.pairs()

    def pairs(self):
        return self._pairs

    def run(self, A, B, C):
        a, b, c = A.numpy(), B.numpy(), C.numpy()
        pair_ptr, a_off, b_off, k = self._pairs
        for t in range(self.n_c):
            m, n = int(self.c_rows[t]), int(self.c_cols[t])
            acc = np.zeros((m, n))
            for p in range(pair_ptr[t], pair_ptr[t + 1]):
                kk = int(k[p])
                acc += a[a_off[p]:a_off[p] + m * kk].reshape(m, kk) @ b[b_off[p]:b_off[p] + kk * n].reshape(kk, n)
            c[self.c_off[t]:self.c_off[t] + m * n] = acc.reshape(-1)


class _FakeSplit:
    """signed 7-bit digit planes of a (rows x k) matrix with row-wise power-of-two scaling, as oz_split_kernel makes them"""

    def __init__(self, mat, slices):
        mx = np.max(np.abs(mat), axis=1) if mat.size else np.zeros(mat.shape[0])
        e = np.where(mx > 0, np.frexp(mx)[1], 0)
        self.scale = np.ldexp(1.0, e)
        if slices <= 9:
            # oz_split_fused_kernel: one conversion to a 64-bit integer, digits peeled off from the least significant end
            xi = np.rint(np.ldexp(mat / self.scale[:, None], 6 + 7 * (slices - 1))).astype(np.int64)
            digs = [None] * slices
            for t in range(slices - 1, 0, -1):
                d = ((xi + 64) & 127) - 64
                xi = (xi - d) >> 7
                digs[t] = d
            digs[0] = xi
            assert np.abs(xi).max(initial=0) <= 64
        else:
            # oz_split_kernel: round to nearest from the most significant end
            v = mat / self.scale[:, None] * 64.0
            digs = []
            for _ in range(slices):
                d = np.rint(v)
                v = (v - d) * 128.0
                digs.append(d.astype(np.int64))
        self.digits = np.array(digs)

    def data_ptr(self):
        return id(self)


def ozaki_product(a, b):
    """A . B^T from two `_FakeSplit` operands (rows of b = columns of the product)"""
    slices = a.digits.shape[0]
    C = np.zeros((a.digits.shape[1], b.digits.shape[1]))
    npass = (slices + 3) // 4
    for g in range(npass - 1, -1, -1):
        d_hi = slices - 1 - 4 * (npass - 1 - g)
        d_lo = max(0, d_hi - 3)
        h = None
        for d in range(d_hi, d_lo - 1, -1):
            Cd = sum(a.digits[t] @ b.digits[d - t].T for t in range(d + 1))
            assert np.abs(Cd).max(initial=0) < 2**31
            h = Cd.astype(np.float64) if h is None else h * 2.0**-7 + Cd
        C += h * 2.0**(-12 - 7 * d_lo) * a.scale[:, None] * b.scale[None, :]
    return C


def _get_block(planes, off, shape):
    """the block at `off` of the device planes (one: real, two: real and imaginary) as a host array"""
    size = int(np.prod(shape))
    blk = planes[0].numpy()[off:off + size]
    if len(planes) == 2:
        blk = blk + 1.j * planes[1].numpy()[off:off + size]
    return blk.reshape(shape)


def _put_block(planes, off, blk):
    """write the host block `blk` at `off` of the device planes (one: real, two: real and imaginary)"""
    for plane, part in zip(planes, (np.real, np.imag)):
        plane.numpy()[off:off + blk.size] = part(blk).reshape(-1)


def _ldexp(blk, e):
    """blk * 2^e, part by part for a complex block"""
    if np.iscomplexobj(blk):
        return np.ldexp(blk.real, e) + 1.j * np.ldexp(blk.imag, e)
    return np.ldexp(blk, e)


def fro_norm(blk):
    """|blk|_F without over- or underflow (the kernels scale every block by a power of two first)"""
    amax = np.max(np.abs(blk), initial=0.)
    return amax * np.linalg.norm(blk / amax) if 0. < amax < np.inf else np.linalg.norm(blk)


class FakeDeviceLib:
    name = 'FAKE numpy test double (tests only)'

    def __init__(self):
        self.torch = torch
        self.c = _lib.load_library()      # host-only entry points of the real library
        self.device = torch.device('cpu')
        self.calls = {}

    def _count(self, name):
        self.calls[name] = self.calls.get(name, 0) + 1

    def stream(self):
        return None

    def _check(self, rc):
        if rc != 0:
            raise _lib.B200Error(self.c.b200_last_error().decode())

    def synchronize(self):
        pass

    def tdot_plan(self, *args):
        self._count('tdot_plan')
        return _FakePlan(_lib.DeviceLib.tdot_plan(self, *args))

    def axpy(self, n, alpha, X, Y):
        self._count('axpy')
        Y.numpy()[:n] += alpha * X.numpy()[:n]

    def scal(self, n, alpha, X):
        self._count('scal')
        X.numpy()[:n] *= alpha

    def dot(self, n, X, Y, scratch, out):
        self._count('dot')
        out.numpy()[0] = float(np.dot(X.numpy()[:n], Y.numpy()[:n]))

    def axpy_segments(self, n_seg, seg_dev, max_len, alpha, X, Y):
        self._count('axpy_segments')
        x, y = X.numpy(), Y.numpy()
        for xo, yo, ln in seg_dev.numpy():
            y[yo:yo + ln] += alpha * x[xo:xo + ln]

    def dot_segments(self, n_seg, seg_dev, max_len, X, Y, scratch, out):
        self._count('dot_segments')
        x, y = X.numpy(), Y.numpy()
        out.numpy()[0] = sum(float(np.dot(x[xo:xo + ln], y[yo:yo + ln])) for xo, yo, ln in seg_dev.numpy())

    def lanczos_update(self, n, alpha, V1, beta, V0, W, scratch, out):
        self._count('lanczos_update')
        w = W.numpy()
        w[:n] -= alpha * V1.numpy()[:n]
        if V0 is not None:
            w[:n] -= beta * V0.numpy()[:n]
        out.numpy()[0] = float(np.dot(w[:n], w[:n]))

    def lanczos_update_dev(self, n, alpha_dev, V1, beta2_dev, V0, W, scratch, out):
        self._count('lanczos_update_dev')
        w = W.numpy()
        w[:n] -= float(alpha_dev.numpy()[0]) * V1.numpy()[:n]
        if V0 is not None and beta2_dev is not None:
            w[:n] -= float(np.sqrt(beta2_dev.numpy()[0])) * V0.numpy()[:n]
        out.numpy()[0] = float(np.dot(w[:n], w[:n]))

    def scal_rsqrt_dev(self, n, norm2_dev, X):
        self._count('scal_rsqrt_dev')
        with np.errstate(divide='ignore', invalid='ignore'):
            X.numpy()[:n] *= 1. / np.sqrt(norm2_dev.numpy()[0])

    def copy_blocks(self, task_host, task_dev, SRC, DST):
        self._count('copy_blocks')
        src, dst = SRC.numpy(), DST.numpy()
        for rec in np.asarray(task_host).reshape(-1, _lib.COPY_REC):
            soff, doff, n, rank = (int(x) for x in rec[:4])
            shape = rec[4:4 + rank]
            ss = rec[4 + _lib.COPY_MAXRANK:4 + _lib.COPY_MAXRANK + rank]
            ds = rec[4 + 2 * _lib.COPY_MAXRANK:4 + 2 * _lib.COPY_MAXRANK + rank]
            assert n == int(np.prod(shape))
            idx = np.indices(tuple(int(s) for s in shape)).reshape(rank, -1)
            so = soff + (idx * ss[:, None]).sum(axis=0)
            do = doff + (idx * ds[:, None]).sum(axis=0)
            dst[do] = src[so]

    def take_blocks(self, task_host, task_dev, idx_dev, SRC, DST):
        self._count('take_blocks')
        src, dst, pool = SRC.numpy(), DST.numpy(), idx_dev.numpy()
        for soff, doff, outer, nk, inner, slen, ioff in np.asarray(task_host).reshape(-1, _lib.TAKE_REC):
            s = src[soff:soff + outer * slen * inner].reshape(outer, slen, inner)
            dst[doff:doff + outer * nk * inner] = s[:, pool[ioff:ioff + nk], :].reshape(-1)

    def scale_axis(self, task_host, task_dev, S_dev, X):
        self._count('scale_axis')
        x, s = X.numpy(), S_dev.numpy()
        for off, outer, ln, inner, soff in np.asarray(task_host).reshape(-1, _lib.SCALE_REC):
            v = x[off:off + outer * ln * inner].reshape(outer, ln, inner)
            v *= s[soff:soff + ln][None, :, None]

    def mid_contract(self, K, N, outer, inner, M, T, OUT):
        self._count('mid_contract')
        m = M.numpy()[:N * K].reshape(N, K)
        t = T.numpy()[:outer * K * inner].reshape(outer, K, inner)
        OUT.numpy()[:outer * N * inner] = np.einsum('nk,oki->oni', m, t).reshape(-1)

    def mid_contract2(self, K1, K2, N1, N2, outer, inner, M, T1, T2, OUT1, OUT2):
        self._count('mid_contract2')
        m = M.numpy()[:(N1 + N2) * (K1 + K2)].reshape(N1 + N2, K1 + K2)
        parts = []
        if K1:
            parts.append(T1.numpy()[:outer * K1 * inner].reshape(outer, K1, inner))
        if K2:
            parts.append(T2.numpy()[:outer * K2 * inner].reshape(outer, K2, inner))
        res = np.einsum('nk,oki->oni', m, np.concatenate(parts, axis=1))
        if N1:
            OUT1.numpy()[:outer * N1 * inner] = res[:, :N1].reshape(-1)
        if N2:
            OUT2.numpy()[:outer * N2 * inner] = res[:, N1:].reshape(-1)

    # -- FP64 products on the int8 tensor path: numpy emulation of the scheme of csrc/ozaki.cu (same digits, exact integer
    #    slice products, diagonals summed in FP64 from the least significant pass)
    def ozaki_split(self, rows, k, X, ld_row, ld_k, slices):
        self._count('ozaki_split')
        x = X.numpy()
        if ld_k == 1:
            mat = np.lib.stride_tricks.as_strided(x, (rows, k), (8 * ld_row, 8)).copy()
        else:
            assert ld_row == 1
            mat = np.lib.stride_tricks.as_strided(x, (rows, k), (8, 8 * ld_k)).copy()
        return _FakeSplit(mat, slices)

    def ozaki_mm(self, m, n, k, slices, a_split, b_split, C, ldc, accumulate=False):
        self._count('ozaki_mm')
        assert a_split.digits.shape == (slices, m, k) and b_split.digits.shape == (slices, n, k)
        res = ozaki_product(a_split, b_split)
        c = np.lib.stride_tricks.as_strided(C.numpy(), (m, n), (8 * ldc, 8))
        if accumulate:
            c += res
        else:
            c[...] = res

    def ozaki_check_abort(self):
        pass

    deflation = True
    deflation_tol = 0.

    def svd_set_deflation_tol(self, tol_rel):
        old, self.deflation_tol = self.deflation_tol, float(tol_rel)
        return old

    def svd_set_deflation(self, on):
        old, self.deflation = self.deflation, bool(on)
        return int(old)

    def block_svd(self, m, n, a_off, u_off, s_off, vt_off, A, U, S, VT):
        self._count('block_svd')
        return self._svd(m, n, a_off, u_off, s_off, vt_off, (A,), (U,), S, (VT,))

    def block_svd_z(self, m, n, a_off, u_off, s_off, vt_off, A_re, A_im, U_re, U_im, S, VT_re, VT_im):
        self._count('block_svd_z')
        return self._svd(m, n, a_off, u_off, s_off, vt_off, (A_re, A_im), (U_re, U_im), S, (VT_re, VT_im))

    def _svd(self, m, n, a_off, u_off, s_off, vt_off, A, U, S, VT):
        """numpy SVD; emulates the kernel's deflation contract: the vectors of the negligible directions are left zero on
        one side.  Real blocks: always rows of VT.  Complex blocks: a block with m >= n is orthogonalised on its columns
        (``transposed`` = 1, zero columns of U), other blocks on their rows (zero rows of VT), so both completion paths
        of ``npc.svd`` run on the CPU."""
        s = S.numpy()
        nact = np.zeros(len(m), dtype=np.int32)
        transp = np.zeros(len(m), dtype=np.int32)
        for i in range(len(m)):
            mi, ni = int(m[i]), int(n[i])
            k = min(mi, ni)
            blk = _get_block(A, a_off[i], (mi, ni))
            uu, ss, vv = np.linalg.svd(blk, full_matrices=False)
            defl = max(16 * 2.220446049250313e-16 * np.sqrt(max(mi, ni)), self.deflation_tol) * fro_norm(blk) \
                if self.deflation else -1.
            r = int(np.sum(ss > defl))
            uu, vv = uu.copy(), vv.copy()
            if len(A) == 2 and mi >= ni:
                transp[i] = 1
                uu[:, r:] = 0.
            else:
                vv[r:] = 0.
            nact[i] = r
            _put_block(U, u_off[i], uu)
            s[s_off[i]:s_off[i] + k] = ss
            _put_block(VT, vt_off[i], vv)
        return np.ones(len(m), dtype=np.int32), nact, transp

    def block_qr(self, m, n, a_off, q_off, r_off, A, Q, R):
        self._count('block_qr')
        self._qr(m, n, a_off, q_off, r_off, (A,), (Q,), (R,))

    def block_qr_z(self, m, n, a_off, q_off, r_off, A_re, A_im, Q_re, Q_im, R_re, R_im):
        self._count('block_qr_z')
        self._qr(m, n, a_off, q_off, r_off, (A_re, A_im), (Q_re, Q_im), (R_re, R_im))

    def _qr(self, m, n, a_off, q_off, r_off, A, Q, R):
        """numpy QR, R with a real non-negative diagonal: the phase (for a real block the sign) of each diagonal entry
        moves into the column of Q.  Like the kernel, it factors 2^-e A, 2^e the power of two of max |a_ij| over both
        planes, and scales R back, so that blocks near the ends of the double range stay finite"""
        for i in range(len(m)):
            blk = _get_block(A, a_off[i], (int(m[i]), int(n[i])))
            mx = max(np.max(np.abs(blk.real), initial=0.), np.max(np.abs(blk.imag), initial=0.))
            e = int(np.clip(np.frexp(mx)[1] - 1, -1022, 1022)) if mx > 0. else 0
            qq, rr = np.linalg.qr(_ldexp(blk, -e))
            d = np.diag(rr)
            ad = np.abs(d)
            safe = np.where(ad > 0., ad, 1.)
            ph = np.where(ad > 0., d.real / safe, 1.)          # part by part: a complex division by a subnormal overflows
            if np.iscomplexobj(d):
                ph = ph + 1.j * (d.imag / safe)
            _put_block(Q, q_off[i], qq * ph[None, :])
            _put_block(R, r_off[i], _ldexp(rr * ph.conj()[:, None], e))

    def col_sqnorms(self, rows, cols, ld, X, OUT):
        self._count('col_sqnorms')
        OUT.numpy()[:cols] = np.sum(X.numpy()[:rows * ld].reshape(rows, ld)[:, :cols]**2, axis=0)

    def grouped_gemm(self, m, n, c_off, pair_ptr, k, a_off, b_off, A, B, C):
        self._count('grouped_gemm')
        a, b, c = A.numpy(), B.numpy(), C.numpy()
        for t in range(len(m)):
            mm, nn = int(m[t]), int(n[t])
            acc = np.zeros((mm, nn))
            for p in range(pair_ptr[t], pair_ptr[t + 1]):
                kk = int(k[p])
                acc += a[a_off[p]:a_off[p] + mm * kk].reshape(mm, kk) @ b[b_off[p]:b_off[p] + kk * nn].reshape(kk, nn)
            c[c_off[t]:c_off[t] + mm * nn] = acc.reshape(-1)

    def block_eigh(self, n, a_off, w_off, v_off, A, W, V):
        self._count('block_eigh')
        return self._eigh(n, a_off, w_off, v_off, (A,), W, (V,))

    def block_eigh_z(self, n, a_off, w_off, v_off, A_re, A_im, W, V_re, V_im):
        self._count('block_eigh_z')
        return self._eigh(n, a_off, w_off, v_off, (A_re, A_im), W, (V_re, V_im))

    def _eigh(self, n, a_off, w_off, v_off, A, W, V):
        """numpy eigh, W ascending, the eigenvectors in the columns of V; like the kernel, a complex block is taken as
        (A + A^H) / 2"""
        w = W.numpy()
        for i in range(len(n)):
            ni = int(n[i])
            blk = _get_block(A, a_off[i], (ni, ni))
            ww, vv = np.linalg.eigh(blk if len(A) == 1 else 0.5 * (blk + blk.conj().T))
            w[w_off[i]:w_off[i] + ni] = ww
            _put_block(V, v_off[i], vv)
        return np.ones(len(n), dtype=np.int32)
