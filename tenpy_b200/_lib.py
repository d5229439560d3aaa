"""ctypes binding of ``libb200npc.so`` (the C ABI declared in ``include/b200npc.h``).

There is exactly one compute backend: the CUDA library built from ``tenpy_b200/csrc`` for sm_90a.
If the shared object is missing, or no CUDA device is visible, every compute entry point raises
:class:`B200Error` -- there is deliberately **no** CPU fallback (the CPU restatement of the path lives
in ``oracle/`` and is test infrastructure only; nothing in this package imports it).

:class:`DeviceLib` is a thin marshalling layer: its methods take ``torch`` tensors (used purely as
device-memory handles) and plain numpy int64 arrays, and forward raw pointers to the C ABI.
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import ctypes
import os

import numpy as np

__all__ = ['B200Error', 'DeviceLib', 'load_library', 'LIB_PATH', 'EXPORTED_SYMBOLS']

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc', 'libb200npc.so')

c_i64p = ctypes.POINTER(ctypes.c_int64)
c_i32p = ctypes.POINTER(ctypes.c_int32)
c_f64p = ctypes.POINTER(ctypes.c_double)
c_vp = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_i32 = ctypes.c_int32
c_f64 = ctypes.c_double

# name -> (restype, argtypes); must list every function declared in include/b200npc.h
_SIGNATURES = {
    'b200_abi_version': (ctypes.c_int, []),
    'b200_last_error': (ctypes.c_char_p, []),
    'b200_device_count': (ctypes.c_int, []),
    'b200_device_info': (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int),
                                        ctypes.POINTER(ctypes.c_int), c_i64p]),
    'b200_kernel_launch_count': (c_i64, [ctypes.c_int]),
    'b200_selftest': (ctypes.c_int, [c_f64p]),
    'b200_find_row_differences': (ctypes.c_int, [c_i64p, c_i64, c_i64, c_i64p, c_i64p]),
    'b200_lexsort_rows': (ctypes.c_int, [c_i64p, c_i64, c_i64, c_i64p]),
    'b200_make_valid': (ctypes.c_int, [c_i64p, c_i64, c_i64, c_i64p]),
    'b200_map_blocks': (ctypes.c_int, [c_i64p, c_i64, c_i64p]),
    'b200_tdot_plan_create': (ctypes.c_int, [c_i64p, c_i64, c_i32, c_i64p, c_i64, c_i32, c_i32, c_i64p, c_i64p,
                                             c_i64p, c_i64p, c_i64p, c_i64p, ctypes.POINTER(c_vp)]),
    'b200_tdot_plan_info': (ctypes.c_int, [c_vp, c_i64p, c_i64p, c_i64p, c_f64p]),
    'b200_tdot_plan_get': (ctypes.c_int, [c_vp, c_i64p, c_i64p, c_i64p, c_i64p]),
    'b200_tdot_plan_pairs': (ctypes.c_int, [c_vp, c_i64p, c_i64p, c_i64p, c_i64p]),
    'b200_tdot_plan_run': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_tdot_plan_destroy': (None, [c_vp]),
    'b200_grouped_gemm_f64': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_i64, c_i64p, c_i64p, c_i64p,
                                             c_vp, c_vp, c_vp, c_vp]),
    'b200_axpy_f64': (ctypes.c_int, [c_i64, c_f64, c_vp, c_vp, c_vp]),
    'b200_scal_f64': (ctypes.c_int, [c_i64, c_f64, c_vp, c_vp]),
    'b200_dot_f64': (ctypes.c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_axpy_segments_f64': (ctypes.c_int, [c_i64, c_vp, c_i64, c_f64, c_vp, c_vp, c_vp]),
    'b200_dot_segments_f64': (ctypes.c_int, [c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_lanczos_update_f64': (ctypes.c_int, [c_i64, c_f64, c_vp, c_f64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_lanczos_update_dev_f64': (ctypes.c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_scal_rsqrt_dev_f64': (ctypes.c_int, [c_i64, c_vp, c_vp, c_vp]),
    'b200_krylov_combine_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_vp, c_i64p, c_vp, c_vp, c_vp]),
    'b200_copy_blocks_f64': (ctypes.c_int, [c_i64, c_vp, c_i64p, c_vp, c_vp, c_vp]),
    'b200_take_blocks_f64': (ctypes.c_int, [c_i64, c_vp, c_i64p, c_vp, c_vp, c_vp, c_vp]),
    'b200_scale_axis_f64': (ctypes.c_int, [c_i64, c_vp, c_i64p, c_vp, c_vp, c_vp]),
    'b200_col_sqnorms_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp]),
    'b200_block_qr_worksize': (c_i64, [c_i64, c_i64p, c_i64p]),
    'b200_block_qr_f64': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    'b200_mid_contract2_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'b200_mid_contract2_z': (ctypes.c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
                                            c_vp, c_vp]),
    'b200_mid_contract_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp]),
    'b200_ozaki_split_worksize': (c_i64, [c_i64, c_i64, c_i32]),
    'b200_ozaki_split_f64': (ctypes.c_int, [c_i64, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp]),
    'b200_ozaki_mm_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp]),
    'b200_ozaki_gemm_worksize': (c_i64, [c_i64, c_i64, c_i64, c_i32]),
    'b200_ozaki_gemm_f64': (ctypes.c_int, [c_i64, c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_i32,
                                           c_vp, c_i64, c_vp]),
    'b200_ozaki_check_abort': (ctypes.c_int, []),
    'b200_svd_set_deflation': (ctypes.c_int, [ctypes.c_int]),
    'b200_svd_set_eig_variant': (ctypes.c_int, [ctypes.c_int]),
    'b200_svd_set_eig_inner_sweeps': (ctypes.c_int, [ctypes.c_int]),
    'b200_svd_set_fused_max_ld': (ctypes.c_int, [ctypes.c_int]),
    'b200_svd_set_deflation_tol': (c_f64, [c_f64]),
    'b200_block_svd_worksize': (c_i64, [c_i64, c_i64p, c_i64p]),
    'b200_block_svd_f64': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp,
                                          c_vp, c_vp, c_i64, c_i32p, c_i32p, c_i32p, c_vp]),
    'b200_block_svd_z_worksize': (c_i64, [c_i64, c_i64p, c_i64p]),
    'b200_block_svd_z': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp, c_vp,
                                        c_vp, c_vp, c_vp, c_vp, c_i64, c_i32p, c_i32p, c_i32p, c_vp]),
    'b200_block_qr_z_worksize': (c_i64, [c_i64, c_i64p, c_i64p]),
    'b200_block_qr_z': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                       c_vp, c_i64, c_vp]),
    'b200_block_eigh_worksize': (c_i64, [c_i64, c_i64p]),
    'b200_block_eigh_f64': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp, c_vp, c_i64,
                                           c_i32p, c_vp]),
    'b200_block_eigh_z_worksize': (c_i64, [c_i64, c_i64p]),
    'b200_block_eigh_z': (ctypes.c_int, [c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                         c_i64, c_i32p, c_vp]),
}
EXPORTED_SYMBOLS = tuple(sorted(_SIGNATURES))

COPY_REC = 22
COPY_MAXRANK = 6
TAKE_REC = 7
SCALE_REC = 5
DOT_SCRATCH = 2048
BLOCK_ALIGN = 16
B200_ERR_NOCONV = 3      # include/b200npc.h


class B200Error(RuntimeError):
    """Raised when the CUDA library is missing or a C-ABI call fails."""


def load_library(path=None):
    """dlopen the C-ABI library and declare all signatures.  Raises B200Error if it is missing."""
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise B200Error("CUDA extension not built: {0} is missing. Run `python -c 'import __graft_entry__ as g; "
                        "g.build()'` (nvcc, sm_90a). tenpy_b200 has no CPU fallback.".format(path))
    try:
        cdll = ctypes.CDLL(path)
    except OSError as e:
        raise B200Error('could not load {0}: {1}'.format(path, e)) from e
    for name, (restype, argtypes) in _SIGNATURES.items():
        try:
            fn = getattr(cdll, name)
        except AttributeError as e:
            raise B200Error('libb200npc.so does not export {0}'.format(name)) from e
        fn.restype = restype
        fn.argtypes = argtypes
    return cdll


def _i64(a):
    a = np.ascontiguousarray(a, dtype=np.int64)
    return a, a.ctypes.data_as(c_i64p)


def _ptr(t):
    """raw device (or host) pointer of a torch tensor / None."""
    if t is None:
        return None
    return c_vp(t.data_ptr())


class _Prof:
    """records a CUDA-event pair around a library call when ``lib.profile`` is a dict (bench / profiling)."""
    __slots__ = ('lib', 'cat', 'ev0', 'info')

    def __init__(self, lib, cat, info=None):
        self.lib, self.cat, self.ev0, self.info = lib, cat, None, info

    def __enter__(self):
        if self.lib.profile is not None:
            self.ev0 = self.lib.torch.cuda.Event(enable_timing=True)
            self.ev0.record()
        return self

    def __exit__(self, *exc):
        if self.ev0 is not None:
            ev1 = self.lib.torch.cuda.Event(enable_timing=True)
            ev1.record()
            self.lib.profile.setdefault(self.cat, []).append((self.ev0, ev1, self.info))
        return False


class TdotPlan:
    """Handle of a contraction plan (``b200_tdot_plan``); see include/b200npc.h."""

    def __init__(self, lib, handle, rank_c):
        self._lib = lib
        self._h = handle
        n_c, n_pairs, c_size = c_i64(), c_i64(), c_i64()
        flops = c_f64()
        lib._check(lib.c.b200_tdot_plan_info(handle, ctypes.byref(n_c), ctypes.byref(n_pairs), ctypes.byref(c_size),
                                             ctypes.byref(flops)))
        self.n_c = n_c.value
        self.n_pairs = n_pairs.value
        self.c_size = c_size.value
        self.flops = flops.value
        self.c_qdata = np.zeros((self.n_c, rank_c), dtype=np.int64)
        self.c_off = np.zeros(self.n_c, dtype=np.int64)
        self.c_rows = np.zeros(self.n_c, dtype=np.int64)
        self.c_cols = np.zeros(self.n_c, dtype=np.int64)
        if self.n_c:
            lib._check(lib.c.b200_tdot_plan_get(handle, self.c_qdata.ctypes.data_as(c_i64p),
                                                self.c_off.ctypes.data_as(c_i64p), self.c_rows.ctypes.data_as(c_i64p),
                                                self.c_cols.ctypes.data_as(c_i64p)))

    def pairs(self):
        """the block-product list: (pair_ptr (n_c+1), a_off, b_off, k) as int64 arrays."""
        lib = self._lib
        pair_ptr = np.zeros(self.n_c + 1, dtype=np.int64)
        a_off = np.zeros(self.n_pairs, dtype=np.int64)
        b_off = np.zeros(self.n_pairs, dtype=np.int64)
        k = np.zeros(self.n_pairs, dtype=np.int64)
        lib._check(lib.c.b200_tdot_plan_pairs(self._h, pair_ptr.ctypes.data_as(c_i64p), a_off.ctypes.data_as(c_i64p),
                                              b_off.ctypes.data_as(c_i64p), k.ctypes.data_as(c_i64p)))
        return pair_ptr, a_off, b_off, k

    def run(self, A, B, C):
        lib = self._lib
        with _Prof(lib, 'gemm', (self.flops, self.n_pairs, self.n_c)):
            lib._check(lib.c.b200_tdot_plan_run(self._h, _ptr(A), _ptr(B), _ptr(C), lib.stream()))

    def __del__(self):
        try:
            if self._h is not None:
                self._lib.c.b200_tdot_plan_destroy(self._h)
                self._h = None
        except Exception:
            pass


class DeviceLib:
    """The (only) compute backend: marshals torch-tensor handles into C-ABI calls."""

    name = 'libb200npc (CUDA sm_90a)'

    def __init__(self, path=None):
        import torch
        self.torch = torch
        self.c = load_library(path)
        if self.c.b200_abi_version() != 1:
            raise B200Error('ABI version mismatch')
        if not torch.cuda.is_available() or self.c.b200_device_count() < 1:
            raise B200Error('no CUDA device visible: tenpy_b200 computes on an H100 only (no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.profile = None   # set to {} to collect CUDA-event timings per kernel family
        self._stream = None
        self.noconv_retries = 0   # block SVD batches repeated with the conservative settings after B200_ERR_NOCONV

    def profile_summary(self):
        """{family: (n_calls, total_ms)} of the collected event pairs; synchronises."""
        self.synchronize()
        out = {}
        for cat, evs in (self.profile or {}).items():
            out[cat] = (len(evs), float(sum(e[0].elapsed_time(e[1]) for e in evs)))
        return out

    def profile_detail(self):
        """{family: [(ms, info), ...]} of the collected event pairs (info: what the call site attached, e.g. the flops
        and the number of block products of a contraction); synchronises."""
        self.synchronize()
        return {cat: [(float(e[0].elapsed_time(e[1])), e[2]) for e in evs] for cat, evs in (self.profile or {}).items()}

    # -- plumbing
    def stream(self):
        """the CUDA stream every kernel of this library handle is enqueued on: torch's current stream at the time of the first
        call (looking it up costs ~10 us of Python per launch, 28 000 times per benchmark sweep); code that switches torch's
        current stream calls :meth:`refresh_stream` afterwards."""
        st = self._stream
        if st is None:
            st = self._stream = c_vp(self.torch.cuda.current_stream().cuda_stream)
        return st

    def refresh_stream(self):
        self._stream = None

    def _check(self, rc):
        if rc != 0:
            msg = self.c.b200_last_error()
            raise B200Error('libb200npc error {0}: {1}'.format(rc, msg.decode() if msg else '?'))

    def synchronize(self):
        self.torch.cuda.current_stream().synchronize()

    # -- tensordot
    def tdot_plan(self, a_qdata, b_qdata, n_contr, a_rows, a_cols, a_off, b_rows, b_cols, b_off):
        a_qdata = np.ascontiguousarray(a_qdata, dtype=np.int64)
        b_qdata = np.ascontiguousarray(b_qdata, dtype=np.int64)
        n_a, rank_a = a_qdata.shape
        n_b, rank_b = b_qdata.shape
        keep = [_i64(x) for x in (a_rows, a_cols, a_off, b_rows, b_cols, b_off)]
        h = c_vp()
        self._check(self.c.b200_tdot_plan_create(a_qdata.ctypes.data_as(c_i64p), n_a, rank_a,
                                                 b_qdata.ctypes.data_as(c_i64p), n_b, rank_b, n_contr, keep[0][1],
                                                 keep[1][1], keep[2][1], keep[3][1], keep[4][1], keep[5][1],
                                                 ctypes.byref(h)))
        return TdotPlan(self, h, rank_a + rank_b - 2 * n_contr)

    def grouped_gemm(self, m, n, c_off, pair_ptr, k, a_off, b_off, A, B, C):
        ms, ns, cs, pp, ks, ao, bo = [_i64(x) for x in (m, n, c_off, pair_ptr, k, a_off, b_off)]
        with _Prof(self, 'gemm'):
            self._check(self.c.b200_grouped_gemm_f64(len(ms[0]), ms[1], ns[1], cs[1], pp[1], len(ks[0]), ks[1], ao[1],
                                                     bo[1], _ptr(A), _ptr(B), _ptr(C), self.stream()))

    # -- FP64 products on the int8 tensor path (csrc/ozaki.cu)
    def ozaki_split(self, rows, k, X, ld_row, ld_k, slices):
        """split a (rows x k) operand (element (r, kk) = X[r*ld_row + kk*ld_k]) into int8 digit planes; returns the
        opaque device buffer (include/b200npc.h)"""
        nbytes = int(self.c.b200_ozaki_split_worksize(int(rows), int(k), int(slices)))
        if nbytes <= 0:
            raise B200Error('ozaki_split: bad shape / slice count')
        out = self.torch.empty(nbytes, dtype=self.torch.uint8, device=self.device)
        with _Prof(self, 'split'):
            self._check(self.c.b200_ozaki_split_f64(int(rows), int(k), _ptr(X), int(ld_row), int(ld_k), int(slices),
                                                    _ptr(out), nbytes, self.stream()))
        return out

    def ozaki_mm(self, m, n, k, slices, a_split, b_split, C, ldc, accumulate=False):
        """C (m x n, ldc) (+)= A . B from two split operands (include/b200npc.h)"""
        with _Prof(self, 'gemm', (2. * m * n * k, 1, 1)):
            self._check(self.c.b200_ozaki_mm_f64(int(m), int(n), int(k), int(slices), _ptr(a_split), _ptr(b_split),
                                                 _ptr(C), int(ldc), 1 if accumulate else 0, self.stream()))

    def ozaki_gemm(self, m, n, k, A, lda, B, ldb, C, ldc, slices, accumulate=False):
        """C (m x n, ldc) (+)= A (m x k, lda) . B (k x n, ldb), all row-major: both splits and the product in one call, the
        digit planes in a workspace allocated here (include/b200npc.h)"""
        nbytes = int(self.c.b200_ozaki_gemm_worksize(int(m), int(n), int(k), int(slices)))
        if nbytes <= 0:
            raise B200Error('ozaki_gemm: bad shape / slice count')
        work = self.torch.empty(nbytes, dtype=self.torch.uint8, device=self.device)
        with _Prof(self, 'gemm', (2. * m * n * k, 1, 1)):
            self._check(self.c.b200_ozaki_gemm_f64(int(m), int(n), int(k), _ptr(A), int(lda), _ptr(B), int(ldb), _ptr(C),
                                                   int(ldc), int(slices), 1 if accumulate else 0, _ptr(work), nbytes,
                                                   self.stream()))

    def ozaki_check_abort(self):
        self._check(self.c.b200_ozaki_check_abort())

    # -- BLAS-1
    def axpy(self, n, alpha, X, Y):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_axpy_f64(n, float(alpha), _ptr(X), _ptr(Y), self.stream()))

    def scal(self, n, alpha, X):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_scal_f64(n, float(alpha), _ptr(X), self.stream()))

    def dot(self, n, X, Y, scratch, out):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_dot_f64(n, _ptr(X), _ptr(Y), _ptr(scratch), _ptr(out), self.stream()))

    def axpy_segments(self, n_seg, seg_dev, max_len, alpha, X, Y):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_axpy_segments_f64(n_seg, _ptr(seg_dev), max_len, float(alpha), _ptr(X), _ptr(Y),
                                                      self.stream()))

    def dot_segments(self, n_seg, seg_dev, max_len, X, Y, scratch, out):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_dot_segments_f64(n_seg, _ptr(seg_dev), max_len, _ptr(X), _ptr(Y), _ptr(scratch),
                                                     _ptr(out), self.stream()))

    def lanczos_update(self, n, alpha, V1, beta, V0, W, scratch, out):
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_lanczos_update_f64(n, float(alpha), _ptr(V1), float(beta), _ptr(V0), _ptr(W),
                                                       _ptr(scratch), _ptr(out), self.stream()))

    def lanczos_update_dev(self, n, alpha_dev, V1, beta2_dev, V0, W, scratch, out):
        """w -= alpha_dev[0] v1 + sqrt(beta2_dev[0]) v0, out[0] = |w|^2: scalars stay on the device"""
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_lanczos_update_dev_f64(n, _ptr(alpha_dev), _ptr(V1), _ptr(beta2_dev), _ptr(V0),
                                                           _ptr(W), _ptr(scratch), _ptr(out), self.stream()))

    def scal_rsqrt_dev(self, n, norm2_dev, X):
        """x *= 1 / sqrt(norm2_dev[0])"""
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_scal_rsqrt_dev_f64(n, _ptr(norm2_dev), _ptr(X), self.stream()))

    def krylov_combine(self, n, in_planes, ptr_host, ptr_dev, coef_dev, OUT):
        """OUT[:2n] = sum_k c_k v_k, c_k = coef_dev[2k] + i coef_dev[2k+1]: `ptr_host` the int64 addresses of the v_k (one
        plane of n or two of 2n doubles, `in_planes`), `ptr_dev` the same table on the device (include/b200npc.h)"""
        ph, php = _i64(ptr_host)
        with _Prof(self, 'blas1'):
            self._check(self.c.b200_krylov_combine_f64(int(n), len(ph), int(in_planes), _ptr(ptr_dev), php,
                                                       _ptr(coef_dev), _ptr(OUT), self.stream()))

    # -- data movement
    def copy_blocks(self, task_host, task_dev, SRC, DST):
        th, thp = _i64(task_host)
        with _Prof(self, 'move'):
            self._check(self.c.b200_copy_blocks_f64(th.shape[0], _ptr(task_dev), thp, _ptr(SRC), _ptr(DST),
                                                    self.stream()))

    def take_blocks(self, task_host, task_dev, idx_dev, SRC, DST):
        th, thp = _i64(task_host)
        with _Prof(self, 'move'):
            self._check(self.c.b200_take_blocks_f64(th.shape[0], _ptr(task_dev), thp, _ptr(idx_dev), _ptr(SRC),
                                                    _ptr(DST), self.stream()))

    def scale_axis(self, task_host, task_dev, S_dev, X):
        th, thp = _i64(task_host)
        with _Prof(self, 'move'):
            self._check(self.c.b200_scale_axis_f64(th.shape[0], _ptr(task_dev), thp, _ptr(S_dev), _ptr(X),
                                                   self.stream()))

    def mid_contract(self, K, N, outer, inner, M, T, OUT):
        """OUT[o, n, i] = sum_k M[n, k] T[o, k, i] (include/b200npc.h)"""
        with _Prof(self, 'move'):
            self._check(self.c.b200_mid_contract_f64(int(K), int(N), int(outer), int(inner), _ptr(M), _ptr(T),
                                                     _ptr(OUT), self.stream()))

    def mid_contract2(self, K1, K2, N1, N2, outer, inner, M, T1, T2, OUT1, OUT2):
        """[OUT1; OUT2][o, n, i] = sum_k M[n, k] [T1; T2][o, k, i] (include/b200npc.h)"""
        with _Prof(self, 'move'):
            self._check(self.c.b200_mid_contract2_f64(int(K1), int(K2), int(N1), int(N2), int(outer), int(inner),
                                                      _ptr(M), _ptr(T1), _ptr(T2), _ptr(OUT1), _ptr(OUT2),
                                                      self.stream()))

    def mid_contract2_z(self, K1, K2, N1, N2, C1, outer, inner, M, T1, T2, OUT1, OUT2):
        """the complex form of :meth:`mid_contract2`: planar M, T1, T2, OUT2; OUT1 the real embedding of
        Y[(o, n / C1), (n % C1, i)] (include/b200npc.h)"""
        with _Prof(self, 'move'):
            self._check(self.c.b200_mid_contract2_z(int(K1), int(K2), int(N1), int(N2), int(C1), int(outer), int(inner),
                                                    _ptr(M), _ptr(T1), _ptr(T2), _ptr(OUT1), _ptr(OUT2),
                                                    self.stream()))

    # -- decompositions
    def _svd_call(self, fn, worksize, m, n, a_off, u_off, s_off, vt_off, A, U, S, VT):
        """one batched block SVD through `fn` (b200_block_svd_f64 or b200_block_svd_z); A, U, VT: tuples of planes.  A batch
        with a block that did not converge within the sweep limit (B200_ERR_NOCONV) runs once more with the conservative
        settings (four inner sweeps of the pivot solver, every direction iterated to convergence) before giving up; A is
        untouched.  Returns (info, nact, transposed)."""
        ms, ns, ao, uo, so, vo = [_i64(x) for x in (m, n, a_off, u_off, s_off, vt_off)]
        nb = len(ms[0])
        wbytes = int(worksize(nb, ms[1], ns[1]))
        work = self.torch.empty(wbytes, dtype=self.torch.uint8, device=self.device)
        info = np.zeros(nb, dtype=np.int32)
        nact = np.zeros(nb, dtype=np.int32)
        transp = np.zeros(nb, dtype=np.int32)
        def call():
            return fn(nb, ms[1], ns[1], ao[1], uo[1], so[1], vo[1], *map(_ptr, A + U + (S,) + VT), _ptr(work), wbytes,
                      info.ctypes.data_as(c_i32p), nact.ctypes.data_as(c_i32p), transp.ctypes.data_as(c_i32p), self.stream())
        with _Prof(self, 'svd'):
            rc = call()
            if rc == B200_ERR_NOCONV:
                self.noconv_retries += 1
                old_in, old_defl = self.svd_set_eig_inner_sweeps(4), self.svd_set_deflation(False)
                try:
                    for t in U + VT:
                        t.zero_()
                    rc = call()
                finally:
                    self.svd_set_eig_inner_sweeps(old_in)
                    self.svd_set_deflation(old_defl)
            self._check(rc)
        return info, nact, transp

    def block_svd(self, m, n, a_off, u_off, s_off, vt_off, A, U, S, VT):
        """batched block SVD (include/b200npc.h); returns (info, nact, transposed)"""
        return self._svd_call(self.c.b200_block_svd_f64, self.c.b200_block_svd_worksize, m, n, a_off, u_off, s_off,
                              vt_off, (A,), (U,), S, (VT,))

    def block_svd_z(self, m, n, a_off, u_off, s_off, vt_off, A_re, A_im, U_re, U_im, S, VT_re, VT_im):
        """complex block SVD on planar buffers (include/b200npc.h); returns (info, nact, transposed) like block_svd"""
        return self._svd_call(self.c.b200_block_svd_z, self.c.b200_block_svd_z_worksize, m, n, a_off, u_off, s_off,
                              vt_off, (A_re, A_im), (U_re, U_im), S, (VT_re, VT_im))

    def _qr_call(self, fn, worksize, m, n, a_off, q_off, r_off, A, Q, R):
        """one batched Householder QR through `fn` (b200_block_qr_f64 or b200_block_qr_z); A, Q, R: tuples of planes"""
        ms, ns, ao, qo, ro = [_i64(x) for x in (m, n, a_off, q_off, r_off)]
        nb = len(ms[0])
        wbytes = int(worksize(nb, ms[1], ns[1]))
        work = self.torch.empty(wbytes, dtype=self.torch.uint8, device=self.device)
        with _Prof(self, 'svd'):
            self._check(fn(nb, ms[1], ns[1], ao[1], qo[1], ro[1], *map(_ptr, A + Q + R), _ptr(work), wbytes,
                           self.stream()))

    def block_qr(self, m, n, a_off, q_off, r_off, A, Q, R):
        """batched Householder QR of the blocks (include/b200npc.h)"""
        self._qr_call(self.c.b200_block_qr_f64, self.c.b200_block_qr_worksize, m, n, a_off, q_off, r_off, (A,), (Q,), (R,))

    def block_qr_z(self, m, n, a_off, q_off, r_off, A_re, A_im, Q_re, Q_im, R_re, R_im):
        """batched complex Householder QR on planar buffers (include/b200npc.h)"""
        self._qr_call(self.c.b200_block_qr_z, self.c.b200_block_qr_z_worksize, m, n, a_off, q_off, r_off, (A_re, A_im),
                      (Q_re, Q_im), (R_re, R_im))

    def col_sqnorms(self, rows, cols, ld, X, OUT):
        with _Prof(self, 'svd'):
            self._check(self.c.b200_col_sqnorms_f64(rows, cols, ld, _ptr(X), _ptr(OUT), self.stream()))

    def svd_set_deflation(self, on):
        return int(self.c.b200_svd_set_deflation(1 if on else 0))

    def svd_set_deflation_tol(self, tol_rel):
        return float(self.c.b200_svd_set_deflation_tol(float(tol_rel)))

    def svd_set_eig_inner_sweeps(self, n):
        """inner sweeps of the version-3 pivot eigen-solver (default 2; 0 = cross mode); returns the old value"""
        return int(self.c.b200_svd_set_eig_inner_sweeps(int(n)))

    def svd_set_fused_max_ld(self, max_ld):
        """row-length limit of the single-launch Jacobi rounds (0: off); returns the old value"""
        return int(self.c.b200_svd_set_fused_max_ld(int(max_ld)))

    def svd_set_eig_variant(self, variant):
        """pivot eigen-solver of the real Jacobi rounds: 1 = jacobi_eig_kernel<false>, 3 = jacobi_eig_kernel_v3 (default);
        other values leave it unchanged (complex rounds always use jacobi_eig_kernel<true>); returns the old value"""
        return int(self.c.b200_svd_set_eig_variant(int(variant)))

    def _eigh_call(self, fn, worksize, prof, n, a_off, w_off, v_off, A, W, V):
        """one batched block eigh through `fn` (b200_block_eigh_f64 or b200_block_eigh_z); A, V: tuples of planes"""
        ns, ao, wo, vo = [_i64(x) for x in (n, a_off, w_off, v_off)]
        nb = len(ns[0])
        wbytes = int(worksize(nb, ns[1]))
        work = self.torch.empty(wbytes, dtype=self.torch.uint8, device=self.device)
        info = np.zeros(nb, dtype=np.int32)
        with _Prof(self, prof):
            self._check(fn(nb, ns[1], ao[1], wo[1], vo[1], *map(_ptr, A + (W,) + V), _ptr(work), wbytes,
                           info.ctypes.data_as(c_i32p), self.stream()))
        return info

    def block_eigh(self, n, a_off, w_off, v_off, A, W, V):
        return self._eigh_call(self.c.b200_block_eigh_f64, self.c.b200_block_eigh_worksize, 'eigh', n, a_off, w_off,
                               v_off, (A,), W, (V,))

    def block_eigh_z(self, n, a_off, w_off, v_off, A_re, A_im, W, V_re, V_im):
        """complex Hermitian block eigh on planar buffers (include/b200npc.h): W real ascending, V unitary; returns info"""
        return self._eigh_call(self.c.b200_block_eigh_z, self.c.b200_block_eigh_z_worksize, 'eigh_z', n, a_off, w_off,
                               v_off, (A_re, A_im), W, (V_re, V_im))

    def kernel_launch_count(self, reset=False):
        return int(self.c.b200_kernel_launch_count(1 if reset else 0))

    def selftest(self):
        out = np.zeros(4, dtype=np.float64)
        self._check(self.c.b200_selftest(out.ctypes.data_as(c_f64p)))
        return out
