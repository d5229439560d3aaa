"""Drop-in replacement of the reference's native module ``tenpy.linalg._npc_helper`` (HOST-buffer plugin).

The reference selects its compiled helper through ``tenpy.tools.optimization.use_cython``
(optimization.py:262-358): at import of ``tenpy.linalg`` every decorated Python function is replaced by
``_npc_helper.__dict__[name]``.  :func:`install` seeds ``sys.modules['tenpy.linalg._npc_helper']`` with THIS
module *before* ``import tenpy`` so that the unmodified reference (its ``Array`` class, DMRG, TEBD ...) calls
into ``libb200npc.so`` through the C ABI:

* the integer helpers (`_make_stride`, `ChargeInfo_make_valid`, `ChargeInfo_check_valid`,
  `LegPipe__init_from_legs`, `_find_row_differences`, `_map_blocks`, `_sliced_copy`,
  `_tensordot_transpose_axes`) run on the host, as they do in the reference's pyx;
* the floating point workers (`_tensordot_worker`, `_inner_worker`, `Array_iadd_prefactor_other`,
  `Array_iscale_prefactor`) take the reference Array's HOST blocks, copy them to the device, run the sm_90a
  kernels and copy the result back (this is the ``e2e`` mode: every call pays PCIe; the device-resident
  mirror ``tenpy_b200.linalg.np_conserved`` is the fast path);
* pure data-movement workers (`Array_itranspose`, `Array__imake_contiguous`, `_combine_legs_worker`,
  `_split_legs_worker`) keep the reference's own Python twins: with host-resident blocks they are numpy views /
  memcpy and nothing is gained by a PCIe round trip.

``use_cython(check_doc=True)`` insists on identical doc strings; they are taken from the reference's source
with ``ast`` (without importing tenpy, which would be circular, SURVEY.md section 8b).
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import ast
import importlib.util
import os
import sys

import numpy as np

compiled_with_MKL = False
QTYPE = np.int64
_charges = None          # set by tenpy.linalg.__init__._patch_cython
_np_conserved = None

_PY_TWINS = {}           # name -> python twin source location (for the functions we do not replace)


def _float_complex_are_64_bit(dtype_float, dtype_complex):
    return np.dtype(dtype_float).itemsize == 8 and np.dtype(dtype_complex).itemsize == 16


def _find_calc_dtype(a_dtype, b_dtype):
    """reference pyx:410: 64-bit float or complex calc dtype and the result dtype"""
    res_dtype = np.promote_types(a_dtype, b_dtype)
    calc = np.promote_types(res_dtype, np.float64)
    return calc, res_dtype


# ------------------------------------------------------------------------------------- integer helpers (host)
def _make_stride(shape, cstyle=True):
    L = len(shape)
    stride = 1
    res = np.empty([L], np.intp)
    if cstyle:
        res[L - 1] = 1
        for a in range(L - 1, 0, -1):
            stride *= shape[a]
            res[a - 1] = stride
    else:
        res[0] = 1
        for a in range(0, L - 1):
            stride *= shape[a]
            res[a + 1] = stride
    return res


def ChargeInfo_make_valid(self, charges=None):
    if charges is None:
        return np.zeros((self.qnumber,), dtype=QTYPE)
    charges = np.array(charges, dtype=QTYPE)
    mod = np.asarray(self._mod)
    mask = mod != 1
    if np.any(mask):
        charges[..., mask] = np.mod(charges[..., mask], mod[mask])
    return charges


def ChargeInfo_check_valid(self, charges):
    charges = np.asarray(charges, dtype=QTYPE)
    mod = np.asarray(self._mod)
    mask = mod != 1
    c = charges[..., mask]
    return bool(np.all(np.logical_and(0 <= c, c < mod[mask])))


def _find_row_differences(qflat):
    if qflat.shape[0] < 2:
        return np.array([0, qflat.shape[0]], dtype=np.intp)
    diff = np.ones(qflat.shape[0] + 1, dtype=np.bool_)
    diff[1:-1] = np.any(qflat[1:] != qflat[:-1], axis=1)
    return np.nonzero(diff)[0]


def _map_blocks(blocksizes):
    return np.repeat(np.arange(len(blocksizes), dtype=np.intp), np.asarray(blocksizes, dtype=np.intp))


def _sliced_copy(dest, dest_beg, src, src_beg, slice_shape):
    if dest_beg is None:
        dest_beg = [0] * dest.ndim
    if src_beg is None:
        src_beg = [0] * src.ndim
    dsl = tuple(slice(int(b), int(b) + int(s)) for b, s in zip(dest_beg, slice_shape))
    ssl = tuple(slice(int(b), int(b) + int(s)) for b, s in zip(src_beg, slice_shape))
    dest[dsl] = src[ssl]


# ------------------------------------------------------------------------------------- floating point workers
def _to_device_array(a):
    """reference Array (host blocks) -> tenpy_b200 Array on the device, same legs tables"""
    from ..linalg import np_conserved as bnpc
    from ..linalg.charges import ChargeInfo, LegCharge
    chinfo = ChargeInfo(list(a.chinfo.mod), list(a.chinfo.names))
    legs = [LegCharge.from_qind(chinfo, l.slices, l.charges, l.qconj) for l in a.legs]
    blocks = [np.ascontiguousarray(b, dtype=np.float64) for b in a._data]
    return bnpc.Array.from_blocks(legs, a._qdata, blocks, a.qtotal)


def _tensordot_worker(a, b, axes):
    if a.dtype.kind == 'c' or b.dtype.kind == 'c':
        raise NotImplementedError('tenpy_b200 shim: real (float64) Arrays only')
    npc = _np_conserved
    from ..linalg import np_conserved as bnpc
    da, db = _to_device_array(a), _to_device_array(b)
    dc = bnpc.tensordot(da, db, axes=axes)
    cut_a = a.rank - axes
    res = npc.Array(a.legs[:cut_a] + b.legs[axes:], np.promote_types(a.dtype, b.dtype),
                    a.chinfo.make_valid(a.qtotal + b.qtotal))
    res._data = dc.get_blocks_host()
    res._qdata = np.array(dc._layout.qdata, dtype=np.intp)
    res._qdata_sorted = True
    return res


def _inner_worker(a, b, do_conj):
    if a.dtype.kind == 'c' or b.dtype.kind == 'c':
        raise NotImplementedError('tenpy_b200 shim: real (float64) Arrays only')
    from ..linalg import np_conserved as bnpc
    da, db = _to_device_array(a), _to_device_array(b)
    return np.float64(bnpc.inner(da, db, axes='range', do_conj=bool(do_conj)))


def Array_iadd_prefactor_other(self, prefactor, other):
    if self.dtype.kind == 'c' or other.dtype.kind == 'c' or isinstance(prefactor, complex):
        raise NotImplementedError('tenpy_b200 shim: real (float64) Arrays only')
    da, db = _to_device_array(self), _to_device_array(other)
    da.iadd_prefactor_other(float(prefactor), db)
    self._data = da.get_blocks_host()
    self._qdata = np.array(da._layout.qdata, dtype=np.intp)
    self._qdata_sorted = True
    return self


def Array_iscale_prefactor(self, prefactor):
    if self.dtype.kind == 'c' or isinstance(prefactor, complex):
        raise NotImplementedError('tenpy_b200 shim: real (float64) Arrays only')
    if prefactor == 0.:
        self._data = []
        self._qdata = np.empty((0, self.rank), np.intp)
        return self
    da = _to_device_array(self)
    da.iscale_prefactor(float(prefactor))
    self._data = da.get_blocks_host()
    self._qdata = np.array(da._layout.qdata, dtype=np.intp)
    self._qdata_sorted = True
    return self


def _svd_worker(a, full_matrices, compute_uv, overwrite_a, cutoff, qtotal_LR, inner_qconj):
    """host-buffer replacement of npc._svd_worker (npc:4950): the per-block LAPACK loop becomes ONE batched
    block-Jacobi call (b200_block_svd_f64).  Installed by :func:`install_workers` (plain assignment, the reference
    looks the worker up by module-global name, npc:3758)."""
    if full_matrices or a.dtype.kind == 'c':
        raise NotImplementedError('tenpy_b200 shim: full_matrices / complex SVD')
    npc = _np_conserved
    from ..linalg import np_conserved as bnpc
    da = _to_device_array(a)
    if not compute_uv:
        S = bnpc.svd(da, compute_uv=False, cutoff=cutoff)
        return None, S, None
    dU, S, dVH = bnpc.svd(da, cutoff=cutoff, qtotal_LR=list(qtotal_LR), inner_qconj=inner_qconj)
    chinfo = a.chinfo
    new_leg_R = npc.LegCharge.from_qind(chinfo, dVH.legs[0].slices, dVH.legs[0].charges, dVH.legs[0].qconj)
    U = npc.Array([a.legs[0], new_leg_R.conj()], a.dtype, dU.qtotal)
    VH = npc.Array([new_leg_R, a.legs[1]], a.dtype, dVH.qtotal)
    U._data, U._qdata, U._qdata_sorted = dU.get_blocks_host(), np.array(dU._layout.qdata, dtype=np.intp), True
    VH._data, VH._qdata, VH._qdata_sorted = dVH.get_blocks_host(), np.array(dVH._layout.qdata, dtype=np.intp), True
    return U, S, VH


def install_workers():
    """after ``import tenpy``: replace the pure-Python LAPACK workers that are not behind `use_cython`."""
    import tenpy.linalg.np_conserved as npc
    npc._svd_worker = _svd_worker
    return npc


# ------------------------------------------------------------------------------------- installation
#: reference function name -> name exported by this module
EXPORTS = ['_make_stride', 'ChargeInfo_make_valid', 'ChargeInfo_check_valid', 'LegPipe__init_from_legs',
           '_find_row_differences', '_map_blocks', '_sliced_copy', 'Array_itranspose', 'Array_iadd_prefactor_other',
           'Array_iscale_prefactor', 'Array__imake_contiguous', '_combine_legs_worker', '_split_legs_worker',
           '_tensordot_transpose_axes', '_tensordot_worker', '_inner_worker']

#: python twins of the reference that are re-used unchanged (compiled from the reference's own source)
_REUSED = {'LegPipe__init_from_legs': ('charges', '_init_from_legs'),
           'Array_itranspose': ('np_conserved', 'itranspose'),
           'Array__imake_contiguous': ('np_conserved', '_imake_contiguous'),
           '_combine_legs_worker': ('np_conserved', '_combine_legs_worker'),
           '_split_legs_worker': ('np_conserved', '_split_legs_worker'),
           '_tensordot_transpose_axes': ('np_conserved', '_tensordot_transpose_axes')}

#: (module, python function name) whose doc string each export has to carry
_DOC_OF = {'_make_stride': ('charges', '_make_stride'), 'ChargeInfo_make_valid': ('charges', 'make_valid'),
           'ChargeInfo_check_valid': ('charges', 'check_valid'), '_find_row_differences': ('charges', '_find_row_differences'),
           '_map_blocks': ('charges', '_map_blocks'), '_sliced_copy': ('charges', '_sliced_copy'),
           'Array_iadd_prefactor_other': ('np_conserved', 'iadd_prefactor_other'),
           'Array_iscale_prefactor': ('np_conserved', 'iscale_prefactor'),
           '_tensordot_worker': ('np_conserved', '_tensordot_worker'), '_inner_worker': ('np_conserved', '_inner_worker')}
_DOC_OF.update(_REUSED)


def _find_defs(tree):
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef,)):
            out.setdefault(node.name, node)
    return out


def install(reference_root=None):
    """Seed ``sys.modules['tenpy.linalg._npc_helper']`` with this module (call BEFORE ``import tenpy``).

    `reference_root`: directory containing the ``tenpy`` package (default: found through ``sys.path``)."""
    if 'tenpy' in sys.modules:
        raise RuntimeError('install() has to be called before tenpy is imported')
    if reference_root is None:
        spec = importlib.util.find_spec('tenpy')
        if spec is None:
            raise ImportError('tenpy not found on sys.path')
        reference_root = os.path.dirname(os.path.dirname(spec.origin))
    me = sys.modules[__name__]
    srcs, trees = {}, {}
    for mod in ('charges', 'np_conserved'):
        path = os.path.join(reference_root, 'tenpy', 'linalg', mod + '.py')
        srcs[mod] = open(path).read()
        trees[mod] = _find_defs(ast.parse(srcs[mod]))
    # re-used python twins: compile the reference's own function source inside a namespace that resolves
    # module globals lazily from the (later injected) reference modules
    for export, (mod, fname) in _REUSED.items():
        node = trees[mod][fname]
        node_src = ast.get_source_segment(srcs[mod], node)
        deco_free = '\n'.join(l for l in node_src.split('\n') if not l.strip().startswith('@use_cython'))
        import textwrap
        code = compile(textwrap.dedent(deco_free), '<tenpy reference %s.%s>' % (mod, fname), 'exec')
        ns = _LazyGlobals(mod)
        exec(code, ns)
        fn = ns[fname]
        fn.__name__ = export
        setattr(me, export, fn)
    for export, (mod, fname) in _DOC_OF.items():
        fn = getattr(me, export)
        fn.__doc__ = ast.get_docstring(trees[mod][fname], clean=False)
    os.environ.pop('TENPY_NO_CYTHON', None)
    sys.modules['tenpy.linalg._npc_helper'] = me
    return me


class _LazyGlobals(dict):
    """globals of a re-used reference function: names are looked up in the reference module once it exists"""

    def __init__(self, modname):
        super().__init__()
        self._modname = modname
        self['__builtins__'] = __builtins__
        self['np'] = np

    def __missing__(self, key):
        mod = sys.modules.get('tenpy.linalg.' + self._modname)
        if mod is not None and hasattr(mod, key):
            return getattr(mod, key)
        other = sys.modules.get('tenpy.linalg.charges')
        if other is not None and hasattr(other, key):
            return getattr(other, key)
        raise KeyError(key)
