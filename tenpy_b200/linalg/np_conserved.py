"""H100-native block-sparse (abelian charge conserving) tensors: the ``np_conserved`` interface.

Host-side mirror of the reference module ``tenpy/linalg/np_conserved.py`` ("npc"): the class
:class:`Array` and the functions :func:`tensordot`, :func:`inner`, :func:`norm`, :func:`svd`,
:func:`eigh`, ... keep the reference's names, argument meaning, label / charge conventions and error
behaviour, so that DMRG code written against ``npc`` reads the same.  The *implementation* is new:

* the blocks of an Array live in ONE packed HBM buffer (:class:`~._layout.BlockLayout`), not in a Python
  list of ndarrays; ``_data`` / ``_qdata`` are materialised on demand for pickling / inspection;
* charge-sector bookkeeping is integer work on the host producing cached *plans*; all floating point
  work is done by the sm_90a kernels of ``libb200npc.so`` (grouped FP64 tensor-core GEMM, BLAS-1 passes
  over the packed buffer, strided block copies, batched block-Jacobi SVD / eigh);
* there is no CPU code path: without the CUDA extension every operation raises ``B200Error``.

Only real (float64) data is supported in this version; the DMRG configurations of the benchmark are
real.  Reference line numbers ("npc:N") refer to tenpy/linalg/np_conserved.py.
"""
# Copyright (C) 2026 tenpy_b200 authors. Apache-2.0.

import itertools
import warnings

import numpy as np

from . import charges
from .charges import ChargeInfo, LegCharge, LegPipe, QTYPE, _lexsort_rows
from ._layout import (BlockLayout, plan_transpose, plan_combine, plan_split, plan_project, plan_scale_axis,
                      plan_take_slice, plan_add_leg, plan_concatenate)
from .. import backend

__all__ = ['QTYPE', 'ChargeInfo', 'LegCharge', 'LegPipe', 'Array', 'zeros', 'eye_like', 'diag', 'tensordot',
           'inner', 'norm', 'svd', 'eigh', 'eigvalsh', 'outer', 'trace', 'to_iterable_arrays', 'pinv', 'concatenate_qdata',
           'concatenate', 'ones', 'detect_qtotal', 'qr']

_PLAN_CACHE = {}
_EMPTY_LAYOUTS = {}      # rank -> the (interned) layout without blocks
_F64 = np.dtype(np.float64)
svd_stats = {'calls': 0, 'jacobi_sweeps': []}   # diagnostics: Jacobi sweeps used by each npc.svd call
_PLAN_CACHE_MAX = 16384


def _conj_label(label):
    """toggle the '*' of a label; pipes '(a.b)' -> '(a*.b*)'."""
    if label is None:
        return None
    if label.startswith('(') and label.endswith(')'):
        return '(' + '.'.join(_conj_label(l) for l in _split_pipe_label(label)) + ')'
    if label.endswith('*'):
        return label[:-1]
    return label + '*'


def _split_pipe_label(label):
    """'(a.(b.c).d)' -> ['a', '(b.c)', 'd']"""
    inner = label[1:-1]
    parts, depth, cur = [], 0, ''
    for ch in inner:
        if ch == '(':
            depth += 1
        elif ch == ')':
            depth -= 1
        if ch == '.' and depth == 0:
            parts.append(cur)
            cur = ''
        else:
            cur += ch
    parts.append(cur)
    return parts


def _allowed_qindices(legs, qtotal, chinfo):
    """All qindex tuples fulfilling the charge rule; (n, rank) int64, lex-sorted."""
    rank = len(legs)
    if rank == 0:
        return np.zeros((1, 0), dtype=np.int64)
    qtotal = chinfo.make_valid(qtotal)
    qd = np.zeros((1, 0), dtype=np.int64)
    part = np.zeros((1, chinfo.qnumber), dtype=QTYPE)
    for ax, leg in enumerate(legs):
        nbk = leg.block_number
        n_old = qd.shape[0]
        qd = np.concatenate([np.repeat(qd, nbk, axis=0), np.tile(np.arange(nbk), n_old)[:, None]], axis=1)
        part = np.repeat(part, nbk, axis=0) + np.tile(leg.charges * leg.qconj, (n_old, 1))
        if ax == rank - 1 and chinfo.qnumber:
            ok = np.all(chinfo.make_valid(part) == qtotal, axis=1)
            qd = qd[ok]
    if qd.shape[0] > 1:
        qd = qd[_lexsort_rows(qd)]
    return qd


class _WriteThroughBlock(np.ndarray):
    """host copy of one stored block; assignments are copied to the device buffer (see :meth:`Array.get_block`)"""
    _target = None

    def __setitem__(self, key, value):
        if np.iscomplexobj(value):
            raise TypeError('a block of a real Array can not hold complex values: assign to the blocks of a '
                            'ComplexArray (.re / .im)')
        np.ndarray.__setitem__(self, key, value)
        if self._target is not None:
            buf, o, s = self._target
            buf[o:o + s].copy_(backend.to_device(np.ascontiguousarray(np.asarray(self), dtype=np.float64).reshape(-1)))

    def __array_finalize__(self, obj):
        self._target = None           # views / results of arithmetic are plain host data


class Array:
    r"""A block-sparse tensor with abelian charge conservation, stored in packed HBM (reference npc:154).

    Parameters
    ----------
    legcharges : list of :class:`LegCharge`
    dtype : only ``np.float64``
    qtotal : total charge (default 0)
    labels : list of {str | None}

    Attributes (as the reference): `rank`, `shape`, `dtype`, `chinfo`, `qtotal`, `legs`, `stored_blocks`,
    `size`; plus `_layout` (the :class:`BlockLayout`) and `_buf` (the device buffer).
    """

    _dtype = _F64

    @property
    def dtype(self):
        return self._dtype

    @dtype.setter
    def dtype(self, dtype):
        """Assigning complex128 to a real Array makes it a :class:`ComplexArray` in place (its blocks become the real
        part), as the reference promotes an Array whose dtype is set (``theta.dtype = ...`` in its ``full_diag_effH``,
        dmrg.py:1207, before complex values are written into a block)."""
        dtype = np.dtype(dtype)
        if dtype.kind == 'c' and not isinstance(self, ComplexArray):
            re = Array.__new__(Array)
            re.__dict__.update(self.__dict__)
            self.__dict__.clear()
            self.__class__ = ComplexArray
            ComplexArray.__init__(self, re, re.zeros_like())
        elif (dtype.kind == 'c') != isinstance(self, ComplexArray):
            raise TypeError('dtype {0} for a ComplexArray: use astype()'.format(dtype))
        else:
            self._dtype = dtype

    def __init__(self, legcharges, dtype=np.float64, qtotal=None, labels=None):
        self.legs = legs = list(legcharges)
        self.rank = rank = len(legs)
        self.shape = tuple([int(l.ind_len) for l in legs])
        if dtype is not np.float64 and np.dtype(dtype) != np.float64:
            raise NotImplementedError('tenpy_b200 supports float64 Arrays only (got {0}); complex tensors: '
                                      'ComplexArray'.format(np.dtype(dtype)))
        self.dtype = _F64
        self.chinfo = chinfo = legs[0].chinfo if rank else ChargeInfo()
        self.qtotal = chinfo.make_valid(qtotal)
        if labels is None:
            self._labels = [None] * rank
        else:
            self._labels = [None] * rank
            self.iset_leg_labels(labels)
        lay = _EMPTY_LAYOUTS.get(rank)
        if lay is None:
            lay = _EMPTY_LAYOUTS[rank] = BlockLayout(np.zeros((0, rank), np.int64), np.zeros((0, rank), np.int64))
        self._layout = lay
        self._buf = None
        self._qdata_sorted = True

    # ------------------------------------------------------------------ basic properties
    def _set_shape(self):
        self.rank = len(self.legs)
        self.shape = tuple(int(l.ind_len) for l in self.legs)

    @property
    def stored_blocks(self):
        return self._layout.nblocks

    @property
    def size(self):
        return int(np.prod(self.shape))

    @property
    def ndim(self):
        return self.rank

    @property
    def _qdata(self):
        return self._layout.qdata.astype(np.intp, copy=False)

    @property
    def _data(self):
        """host copies of the blocks (list of ndarrays); synchronises."""
        return self.get_blocks_host()

    def get_blocks_host(self):
        lay = self._layout
        if lay.nblocks == 0:
            return []
        host = backend.to_host(self._buf)
        return [host[o:o + s].reshape(sh).copy() for o, s, sh in zip(lay.offsets, lay.sizes, lay.shapes)]

    def _set_blocks(self, layout, buf):
        self._layout = layout
        self._buf = buf
        return self

    def test_sanity(self):
        """Consistency checks (reference npc:223)."""
        if len(self.legs) != self.rank or len(self._labels) != self.rank:
            raise ValueError('wrong number of legs/labels')
        for leg in self.legs:
            if leg.chinfo != self.chinfo:
                raise ValueError('leg with different ChargeInfo')
        lay = self._layout
        if lay.rank != self.rank:
            raise ValueError('layout rank mismatch')
        if lay.nblocks:
            if self._buf is None or self._buf.numel() != lay.size:
                raise ValueError('buffer size mismatch')
            for ax, leg in enumerate(self.legs):
                if np.any(lay.qdata[:, ax] >= leg.block_number) or np.any(lay.qdata[:, ax] < 0):
                    raise ValueError('qindex out of range')
                if np.any(leg.get_block_sizes()[lay.qdata[:, ax]] != lay.shapes[:, ax]):
                    raise ValueError('block shape mismatch')
            part = np.zeros((lay.nblocks, self.chinfo.qnumber), dtype=QTYPE)
            for ax, leg in enumerate(self.legs):
                part += leg.charges[lay.qdata[:, ax]] * leg.qconj
            if np.any(self.chinfo.make_valid(part) != self.qtotal):
                raise ValueError('block violates the charge rule')

    # ------------------------------------------------------------------ construction
    def copy(self, deep=True):
        """Copy; ``deep=False`` shares the device buffer (reference npc:272)."""
        res = Array.__new__(Array)
        res.__dict__.update(self.__dict__)
        res.legs = list(self.legs)
        res._labels = list(self._labels)
        res.qtotal = self.qtotal.copy()
        if deep and self._buf is not None:
            res._buf = self._buf.clone()
        return res

    def __getstate__(self):
        d = dict(self.__dict__)
        lay = self._layout
        d['_buf'] = None if self._buf is None else backend.to_host(self._buf)
        d['_layout'] = (lay.qdata, lay.shapes)
        return d

    def __setstate__(self, state):
        qd, sh = state.pop('_layout')
        host = state.pop('_buf')
        self.__dict__.update(state)
        self._layout = BlockLayout(qd, sh)
        self._buf = None if host is None else backend.to_device(host)

    @classmethod
    def from_blocks(cls, legcharges, qdata, blocks, qtotal=None, labels=None):
        """Create from host blocks: `qdata` (n, rank) qindices, `blocks` list of ndarrays."""
        if cls is Array and any(np.iscomplexobj(b) for b in blocks):
            return ComplexArray.from_blocks(legcharges, qdata, blocks, qtotal, labels)
        res = cls(legcharges, np.float64, qtotal, labels)
        qdata = np.asarray(qdata, dtype=np.int64).reshape(-1, res.rank)
        layout, perm = BlockLayout.from_legs(res.legs, qdata)
        host = np.zeros(layout.size, dtype=np.float64)
        for new_i, old_i in enumerate(perm):
            blk = np.asarray(blocks[old_i], dtype=np.float64)
            if tuple(blk.shape) != tuple(layout.shapes[new_i]):
                raise ValueError('block {0} has shape {1}, expected {2}'.format(old_i, blk.shape,
                                                                               tuple(layout.shapes[new_i])))
            o = layout.offsets[new_i]
            host[o:o + layout.sizes[new_i]] = blk.reshape(-1)
        res._set_blocks(layout, backend.to_device(host))
        return res

    @classmethod
    def from_device_buffer(cls, legcharges, qdata, buf, qtotal=None, labels=None):
        """Wrap an existing packed device buffer (`qdata` must be lex-sorted; `buf` laid out as BlockLayout)."""
        res = cls(legcharges, np.float64, qtotal, labels)
        layout, perm = BlockLayout.from_legs(res.legs, qdata)
        if np.any(perm != np.arange(len(perm))):
            raise ValueError('qdata has to be lex-sorted')
        if buf.numel() != layout.size:
            raise ValueError('buffer has {0} elements, layout needs {1}'.format(buf.numel(), layout.size))
        return res._set_blocks(layout, buf)

    @classmethod
    def from_ndarray_trivial(cls, data_flat, dtype=None, labels=None):
        """Array without charges from a dense ndarray (reference npc:420)."""
        if np.iscomplexobj(data_flat) or (dtype is not None and np.dtype(dtype).kind == 'c'):
            data_flat = np.asarray(data_flat)
            chinfo = ChargeInfo()
            return ComplexArray.from_ndarray(data_flat, [LegCharge.from_trivial(s, chinfo) for s in data_flat.shape],
                                             labels=labels)
        data_flat = np.asarray(data_flat, dtype=np.float64)
        chinfo = ChargeInfo()
        legs = [LegCharge.from_trivial(s, chinfo) for s in data_flat.shape]
        return cls.from_blocks(legs, np.zeros((1, data_flat.ndim), np.int64), [data_flat], None, labels)

    @classmethod
    def from_ndarray(cls, data_flat, legcharges, dtype=None, qtotal=None, cutoff=None, labels=None,
                     raise_wrong_sector=True, warn_wrong_sector=True):
        """Dense ndarray -> Array, keeping blocks with an entry ``> cutoff`` (reference npc:451)."""
        if cutoff is None:
            cutoff = 1e-16
        if cls is Array and (np.iscomplexobj(data_flat) or (dtype is not None and np.dtype(dtype).kind == 'c')):
            return ComplexArray.from_ndarray(data_flat, legcharges, dtype, qtotal, cutoff, labels, raise_wrong_sector,
                                             warn_wrong_sector)
        data_flat = np.asarray(data_flat, dtype=np.float64)
        legcharges = list(legcharges)
        if data_flat.shape != tuple(l.ind_len for l in legcharges):
            raise ValueError('shape mismatch: {0} vs legs {1}'.format(data_flat.shape,
                                                                      tuple(l.ind_len for l in legcharges)))
        chinfo = legcharges[0].chinfo
        if qtotal is None:
            qtotal = cls.detect_qtotal(data_flat, legcharges, cutoff)
        qd_all = _allowed_qindices(legcharges, qtotal, chinfo)
        qd, blocks = [], []
        covered = np.zeros(data_flat.shape, dtype=np.bool_) if (raise_wrong_sector or warn_wrong_sector) else None
        for row in qd_all:
            sl = tuple(l.get_slice(qi) for l, qi in zip(legcharges, row))
            blk = data_flat[sl]
            if covered is not None:
                covered[sl] = True
            if np.any(np.abs(blk) > cutoff):
                qd.append(row)
                blocks.append(blk)
        if covered is not None and np.any(np.abs(data_flat[~covered]) > cutoff):
            if raise_wrong_sector:
                raise ValueError('wrong sector with non-zero entries')
            warnings.warn('flat array has non-zero entries in blocks incompatible with charge', stacklevel=2)
        qd = np.array(qd, dtype=np.int64).reshape(-1, len(legcharges))
        return cls.from_blocks(legcharges, qd, blocks, qtotal, labels)

    @staticmethod
    def detect_qtotal(flat_array, legcharges, cutoff=None):
        """Total charge of the largest entry (reference npc:603)."""
        if cutoff is None:
            cutoff = 1e-16
        flat_array = np.asarray(flat_array)
        inds = np.unravel_index(np.argmax(np.abs(flat_array)), flat_array.shape)
        chinfo = legcharges[0].chinfo
        tot = np.zeros(chinfo.qnumber, dtype=QTYPE)
        for leg, i in zip(legcharges, inds):
            qi, _ = leg.get_qindex(int(i))
            tot += leg.get_charge(qi)
        return chinfo.make_valid(tot)

    @classmethod
    def from_func(cls, func, legcharges, dtype=None, qtotal=None, func_args=(), func_kwargs={}, shape_kw=None,
                  labels=None):
        """Fill all charge-allowed blocks with ``func(shape)`` (reference npc:617).  Complex blocks give a
        :class:`ComplexArray`, as in :meth:`from_blocks`."""
        legcharges = list(legcharges)
        chinfo = legcharges[0].chinfo
        qd = _allowed_qindices(legcharges, qtotal, chinfo)
        blocks = []
        for row in qd:
            shape = tuple(int(l.get_block_sizes()[qi]) for l, qi in zip(legcharges, row))
            if shape_kw is None:
                blk = func(shape, *func_args, **func_kwargs)
            else:
                kw = dict(func_kwargs)
                kw[shape_kw] = shape
                blk = func(*func_args, **kw)
            blk = np.asarray(blk)
            blocks.append((blk if np.iscomplexobj(blk) else blk.astype(np.float64, copy=False)).reshape(shape))
        return cls.from_blocks(legcharges, qd, blocks, qtotal, labels)

    def zeros_like(self):
        res = self.copy(deep=False)
        res._layout = BlockLayout(np.zeros((0, self.rank), np.int64), np.zeros((0, self.rank), np.int64))
        res._buf = None
        return res

    def to_ndarray(self):
        """Dense host ndarray (reference npc:890); synchronises."""
        res = np.zeros(self.shape, dtype=np.float64)
        lay = self._layout
        if lay.nblocks:
            host = backend.to_host(self._buf)
            for qi, o, s, sh in zip(lay.qdata, lay.offsets, lay.sizes, lay.shapes):
                sl = tuple(l.get_slice(q) for l, q in zip(self.legs, qi))
                res[sl] = host[o:o + s].reshape(sh)
        return res

    def get_block(self, qindices, insert=False, raise_incomp_q=False):
        """The block with given qindices as a host array, or None (reference npc:1330).  The reference hands out a view
        of its host block; here the result is a host copy whose item assignments are written through to the device buffer
        (``block[:] = values`` as in the reference's ``full_diag_effH``, dmrg.py:1209).  ``insert=True`` stores a zero
        block first if there is none."""
        qindices = np.asarray(qindices, dtype=np.int64)
        lay = self._layout
        match = np.nonzero(np.all(lay.qdata == qindices, axis=1))[0]
        if len(match) == 0:
            if not insert:
                return None
            part = np.zeros(self.chinfo.qnumber, dtype=QTYPE)
            for leg, qi in zip(self.legs, qindices):
                part = part + leg.get_charge(int(qi)) * leg.qconj
            if np.any(self.chinfo.make_valid(part) != self.qtotal):
                if raise_incomp_q:
                    raise ValueError('trying to get block for incompatible charges')
                return None
            shape = tuple(int(leg.get_block_sizes()[int(qi)]) for leg, qi in zip(self.legs, qindices))
            new = Array.from_blocks(self.legs, np.concatenate([lay.qdata, qindices[None, :]], axis=0),
                                    self.get_blocks_host() + [np.zeros(shape)], self.qtotal, self._labels)
            self._layout, self._buf = new._layout, new._buf
            lay = self._layout
            match = np.nonzero(np.all(lay.qdata == qindices, axis=1))[0]
        i = int(match[0])
        o, s = int(lay.offsets[i]), int(lay.sizes[i])
        host = backend.to_host(self._buf[o:o + s]).reshape(lay.shapes[i]).view(_WriteThroughBlock)
        host._target = (self._buf, o, s)
        return host

    # ------------------------------------------------------------------ labels
    def get_leg_index(self, label):
        if isinstance(label, str):
            try:
                return self._labels.index(label)
            except ValueError:
                raise KeyError('label not found: ' + repr(label) + ', current labels ' +
                               repr(self.get_leg_labels())) from None
        label = int(label)
        if label < 0:
            label += self.rank
        if not 0 <= label < self.rank:
            raise ValueError('axis out of range')
        return label

    def get_leg_indices(self, labels):
        return [self.get_leg_index(l) for l in labels]

    def iset_leg_labels(self, labels):
        labels = list(labels)
        if len(labels) != self.rank:
            raise ValueError('need one label per leg')
        seen = [l for l in labels if l is not None]
        if len(seen) != len(set(seen)):
            raise ValueError('duplicate label in ' + repr(labels))
        self._labels = [None if l is None else str(l) for l in labels]
        return self

    def get_leg_labels(self):
        return list(self._labels)

    def has_label(self, label):
        return label in self._labels

    def get_leg(self, label):
        return self.legs[self.get_leg_index(label)]

    def ireplace_label(self, old_label, new_label):
        ax = self.get_leg_index(old_label)
        labels = list(self._labels)
        labels[ax] = None
        if new_label is not None and new_label in labels:
            raise ValueError('duplicate label ' + repr(new_label))
        labels[ax] = new_label
        self._labels = labels
        return self

    def replace_label(self, old_label, new_label):
        return self.copy(deep=False).ireplace_label(old_label, new_label)

    def ireplace_labels(self, old_labels, new_labels):
        axes = self.get_leg_indices(old_labels)
        labels = list(self._labels)
        for ax in axes:
            labels[ax] = None
        for ax, nl in zip(axes, new_labels):
            if nl is not None and nl in labels:
                raise ValueError('duplicate label ' + repr(nl))
            labels[ax] = nl
        self._labels = labels
        return self

    def replace_labels(self, old_labels, new_labels):
        return self.copy(deep=False).ireplace_labels(old_labels, new_labels)

    def idrop_labels(self, old_labels=None):
        if old_labels is None:
            self._labels = [None] * self.rank
        else:
            for ax in self.get_leg_indices(old_labels):
                self._labels[ax] = None
        return self

    # ------------------------------------------------------------------ conj / transpose
    def iconj(self, complex_conj=True):
        """Conjugate: flip all legs and the total charge, toggle '*' of labels (reference npc:2035)."""
        self.qtotal = self.chinfo.make_valid(-self.qtotal)
        self.legs = [l.conj() for l in self.legs]
        self._labels = [_conj_label(l) for l in self._labels]
        return self

    def conj(self, complex_conj=True):
        return self.copy(deep=False).iconj(complex_conj)

    def _parse_axes(self, axes):
        if axes is None:
            return list(reversed(range(self.rank)))
        axes = self.get_leg_indices(list(axes))
        if len(axes) != self.rank or sorted(axes) != list(range(self.rank)):
            raise ValueError('axes has wrong length / is not a permutation: ' + repr(axes))
        return axes

    def itranspose(self, axes=None):
        """Transpose in place (reference npc:2057); blocks are physically permuted on the device."""
        axes = self._parse_axes(axes)
        if axes == list(range(self.rank)):
            return self
        old_layout = self._layout
        self.legs = [self.legs[a] for a in axes]
        self._labels = [self._labels[a] for a in axes]
        self._set_shape()
        key = ('T', tuple(axes))
        cached = old_layout.cache.get(key)
        if cached is None:
            new_layout, rec = plan_transpose(old_layout, axes)
            cached = (new_layout, rec, backend.to_device(rec) if len(rec) else None)
            old_layout.cache[key] = cached
        new_layout, rec, rec_dev = cached
        if old_layout.nblocks:
            buf = _dest_buffer(new_layout, rec)
            backend.get_lib().copy_blocks(rec, rec_dev, self._buf, buf)
            self._buf = buf
        self._layout = new_layout
        return self

    def transpose(self, axes=None):
        return self.copy(deep=False).itranspose(axes)

    # ------------------------------------------------------------------ elementwise
    def _binary_same_layout(self, other):
        return self._layout.same_blocks(other._layout)

    def iscale_prefactor(self, prefactor):
        """``self *= prefactor`` (reference npc:2386 / pyx:964)."""
        if self._layout.nblocks:
            if prefactor == 0.0:
                self._layout = BlockLayout(np.zeros((0, self.rank), np.int64), np.zeros((0, self.rank), np.int64))
                self._buf = None
            else:
                backend.get_lib().scal(self._layout.size, prefactor, self._buf)
        return self

    def iadd_prefactor_other(self, prefactor, other):
        """``self += prefactor * other`` (reference npc:2373 / pyx:860).  A real Array can not become complex in place:
        a complex `prefactor` or a :class:`ComplexArray` `other` raises TypeError (``self + prefactor * other`` gives
        the ComplexArray)."""
        if isinstance(other, ComplexArray) or isinstance(prefactor, (complex, np.complexfloating)):
            raise TypeError('iadd_prefactor_other of a real Array with a complex prefactor or a ComplexArray: use the '
                            'out-of-place form self + prefactor * other')
        if self.rank != other.rank or self.shape != other.shape:
            raise ValueError('incompatible shapes {0} vs {1}'.format(self.shape, other.shape))
        if np.any(self.qtotal != other.qtotal):
            raise ValueError('Arrays can not be added: different qtotal')
        other = other._match_labels_of(self)
        for ls, lo in zip(self.legs, other.legs):
            ls.test_equal(lo)
        if other._layout.nblocks == 0 or prefactor == 0.0:
            return self
        lib = backend.get_lib()
        if self._layout.nblocks == 0:
            self._layout = other._layout
            self._buf = other._buf.clone()
            lib.scal(self._layout.size, prefactor, self._buf)
            return self
        if self._binary_same_layout(other):
            lib.axpy(self._layout.size, prefactor, other._buf, self._buf)
            return self
        # different block tables: move self into the union layout, then add segment-wise
        a, b = self._layout, other._layout
        union, seg_self, seg_other = _union_layout(self.legs, a, b)
        buf = backend.zeros(union.size)
        if len(seg_self):
            lib.axpy_segments(len(seg_self), backend.to_device(seg_self), int(seg_self[:, 2].max()), 1.0, self._buf,
                              buf)
        lib.axpy_segments(len(seg_other), backend.to_device(seg_other), int(seg_other[:, 2].max()), prefactor,
                          other._buf, buf)
        self._layout, self._buf = union, buf
        return self

    def _match_labels_of(self, ref):
        """transpose `self` such that its labels are in the order of `ref` (if both are fully labelled)."""
        if self._labels == ref._labels:
            return self
        if None in self._labels or None in ref._labels or set(self._labels) != set(ref._labels):
            return self
        return self.transpose(ref._labels)

    def __mul__(self, other):
        if np.iscomplexobj(other) and np.isscalar(other):     # real Array * complex scalar: a ComplexArray
            z = complex(other)
            return ComplexArray(self.copy(deep=True).iscale_prefactor(z.real), self.copy(deep=True).iscale_prefactor(z.imag))
        if np.isscalar(other):
            return self.copy(deep=True).iscale_prefactor(float(other))
        return NotImplemented

    __rmul__ = __mul__

    def __imul__(self, other):
        if np.iscomplexobj(other) and np.isscalar(other):     # changes the type: ``a *= z`` rebinds `a`
            return self.__mul__(other)
        if np.isscalar(other):
            return self.iscale_prefactor(float(other))
        return NotImplemented

    def __truediv__(self, other):
        if np.isscalar(other):
            return self.__mul__(1.0 / other)
        return NotImplemented

    def __itruediv__(self, other):
        if np.iscomplexobj(other) and np.isscalar(other):
            return self.__mul__(1.0 / other)
        if np.isscalar(other):
            return self.iscale_prefactor(1.0 / other)
        return NotImplemented

    def __neg__(self):
        return self.__mul__(-1.0)

    def __add__(self, other):
        if isinstance(other, Array):
            return self.copy(deep=True).iadd_prefactor_other(1.0, other)
        return NotImplemented

    def __iadd__(self, other):
        if isinstance(other, Array):
            return self.iadd_prefactor_other(1.0, other)
        return NotImplemented

    def __sub__(self, other):
        if isinstance(other, Array):
            return self.copy(deep=True).iadd_prefactor_other(-1.0, other)
        return NotImplemented

    def __isub__(self, other):
        if isinstance(other, Array):
            return self.iadd_prefactor_other(-1.0, other)
        return NotImplemented

    def norm(self, ord=None, convert_to_float=True):
        """Frobenius norm (reference npc:2241)."""
        if ord not in (None, 2, 'fro'):
            raise NotImplementedError('only the 2-norm is implemented')
        if self._layout.nblocks == 0:
            return 0.0
        lib = backend.get_lib()
        out = backend.scalar_out()
        lib.dot(self._layout.size, self._buf, self._buf, backend.dot_scratch(), out)
        return float(np.sqrt(backend.read_scalar(out)))

    def astype(self, dtype, copy=True):
        """float64: a copy; complex128: a :class:`ComplexArray` with this Array as real part and no imaginary blocks."""
        if np.dtype(dtype) == np.complex128:
            return ComplexArray(self.copy(deep=True), self.zeros_like())
        if np.dtype(dtype) != np.float64:
            raise NotImplementedError('Arrays are float64 or complex128 (ComplexArray), not {0}'.format(np.dtype(dtype)))
        return self.copy(deep=copy)

    # ------------------------------------------------------------------ scale_axis / project
    def iscale_axis(self, s, axis=-1):
        """Multiply slice ``i`` along `axis` by ``s[i]`` (reference npc:2108).  A real Array can not become complex in
        place: `s` with a non-zero imaginary part raises TypeError (:meth:`scale_axis` returns the ComplexArray)."""
        axis = self.get_leg_index(axis)
        if np.iscomplexobj(s):
            s = np.asarray(s)
            if np.any(s.imag != 0.):
                raise TypeError('iscale_axis of a real Array with complex factors: use scale_axis, which returns a '
                                'ComplexArray')
            s = s.real
        s = np.asarray(s, dtype=np.float64)
        if s.shape != (self.shape[axis],):
            raise ValueError('s has wrong shape {0}, expected ({1},)'.format(s.shape, self.shape[axis]))
        lay = self._layout
        if lay.nblocks == 0:
            return self
        key = ('S', axis, self.legs[axis].slices.tobytes())
        cached = lay.cache.get(key)
        if cached is None:
            rec = plan_scale_axis(lay, self.legs[axis], axis)
            cached = (rec, backend.to_device(rec))
            lay.cache[key] = cached
        rec, rec_dev = cached
        backend.get_lib().scale_axis(rec, rec_dev, backend.to_device(s), self._buf)
        return self

    def scale_axis(self, s, axis=-1):
        """Copy of `self` with slice ``i`` along `axis` multiplied by ``s[i]``; complex `s` gives a ComplexArray."""
        if np.iscomplexobj(s):
            s = np.asarray(s)
            return ComplexArray(self.scale_axis(s.real, axis), self.scale_axis(s.imag, axis))
        return self.copy(deep=True).iscale_axis(s, axis)

    def iproject(self, mask, axes):
        """Keep only the indices selected by `mask` along `axes` (reference npc:1914).

        Returns ``(map_qind, block_masks)`` of the (last) projected leg, like the reference."""
        if not isinstance(axes, (list, tuple)):
            axes = [axes]
            mask = [mask]
        out = (None, None)
        for m, ax in zip(mask, axes):
            ax = self.get_leg_index(ax)
            m = np.asarray(m)
            if m.dtype != np.bool_:
                full = np.zeros(self.shape[ax], dtype=np.bool_)
                full[m] = True
                m = full
            if m.shape != (self.shape[ax],):
                raise ValueError('mask has wrong length')
            leg = self.legs[ax]
            lay = self._layout
            key = ('J', ax, leg.content_key(), m.tobytes())
            cached = lay.cache.get(key)
            if cached is None:
                map_qind, block_masks, new_leg = leg.project(m)
                new_legs_ = list(self.legs)
                new_legs_[ax] = new_leg
                new_layout, rec, pool = plan_project(lay, self.legs, ax, map_qind, block_masks, new_leg, new_legs_)
                cached = (map_qind, block_masks, new_leg, new_layout, rec,
                          backend.to_device(rec) if new_layout.nblocks else None,
                          backend.to_device(pool) if new_layout.nblocks else None)
                if len(lay.cache) < 256:
                    lay.cache[key] = cached
            map_qind, block_masks, new_leg, new_layout, rec, rec_dev, pool_dev = cached
            new_legs = list(self.legs)
            new_legs[ax] = new_leg
            if new_layout.nblocks:
                buf = backend.zeros(new_layout.size)
                backend.get_lib().take_blocks(rec, rec_dev, pool_dev, self._buf, buf)
            else:
                buf = None
            self.legs = new_legs
            self._set_shape()
            self._layout, self._buf = new_layout, buf
            out = (map_qind, block_masks)
        return out

    # ------------------------------------------------------------------ pipes
    def make_pipe(self, axes, **kwargs):
        """LegPipe for the given axes (reference npc:1541)."""
        axes = self.get_leg_indices(axes)
        legs = [self.legs[a] for a in axes]
        kwargs.setdefault('qconj', legs[0].qconj)
        return LegPipe(legs, **kwargs)

    def combine_legs(self, combine_legs, new_axes=None, pipes=None, qconj=None, _view=False):
        """Reshape: fuse bundles of legs into pipes (reference npc:1561; worker npc:4404 / pyx:1013).

        ``_view=True`` (internal): if the move is a pure relabelling of the packed buffer, share it instead of
        copying -- only for callers that own `self` or treat the result as read-only."""
        combine_legs = list(combine_legs)
        if len(combine_legs) and not isinstance(combine_legs[0], (list, tuple, np.ndarray)):
            combine_legs = [combine_legs]
        combine_legs = [self.get_leg_indices(cl) for cl in combine_legs]
        flat = [a for cl in combine_legs for a in cl]
        if len(set(flat)) != len(flat):
            raise ValueError('an axis appears twice in combine_legs')
        npipes = len(combine_legs)
        # default new axes: position of the first leg of each bundle, accounting for removed legs
        if new_axes is None:
            new_axes = []
            for cl in combine_legs:
                first = cl[0]
                removed = sum(1 for c2 in combine_legs for a in c2[1:] if a < first)
                new_axes.append(first - removed)
        else:
            new_axes = list(np.atleast_1d(new_axes))
            new_rank = self.rank - len(flat) + npipes
            new_axes = [a + new_rank if a < 0 else a for a in new_axes]
        if len(set(new_axes)) != npipes:
            raise ValueError('new_axes not unique')
        if pipes is None:
            pipes = [None] * npipes
        elif isinstance(pipes, LegPipe):
            pipes = [pipes]
        if qconj is None:
            qconj = [None] * npipes
        else:
            qconj = list(np.atleast_1d(qconj))
        pipes = list(pipes)
        for j, cl in enumerate(combine_legs):
            if pipes[j] is None:
                qc = qconj[j] if qconj[j] is not None else self.legs[cl[0]].qconj
                pipes[j] = self.make_pipe(cl, qconj=qc)
            else:
                pipe = pipes[j]
                if pipe.nlegs != len(cl):
                    raise ValueError('pipe has wrong number of legs')
                legs = [self.legs[a] for a in cl]
                if legs[0].qconj != pipe.legs[0].qconj:
                    pipes[j] = pipe = pipe.conj()
                for l1, l2 in zip(legs, pipe.legs):
                    l1.test_equal(l2)
        # sort by new_axes (ascending), as the worker expects
        order = np.argsort(new_axes)
        combine_legs = [combine_legs[i] for i in order]
        pipes = [pipes[i] for i in order]
        new_axes = [int(new_axes[i]) for i in order]
        non_combined = [a for a in range(self.rank) if a not in flat]
        new_rank = len(non_combined) + npipes
        non_new_axes = [a for a in range(new_rank) if a not in new_axes]
        res_legs = [None] * new_rank
        res_labels = [None] * new_rank
        for na, pipe, cl in zip(new_axes, pipes, combine_legs):
            res_legs[na] = pipe
            sub = [self._labels[a] for a in cl]
            res_labels[na] = None if None in sub else '(' + '.'.join(sub) + ')'
        for na, oa in zip(non_new_axes, non_combined):
            res_legs[na] = self.legs[oa]
            res_labels[na] = self._labels[oa]
        res = Array(res_legs, self.dtype, self.qtotal, res_labels)
        lay = self._layout
        if lay.nblocks == 0:
            return res
        key = ('C', tuple(tuple(cl) for cl in combine_legs), tuple(new_axes), tuple(p.content_key() for p in pipes))
        cached = lay.cache.get(key)
        if cached is None:
            new_layout, rec = plan_combine(lay, self.legs, combine_legs, new_axes, pipes, res_legs)
            cached = (new_layout, rec, backend.to_device(rec), pipes)
            lay.cache[key] = cached
        new_layout, rec, rec_dev = cached[:3]
        if _view and new_layout.size == lay.size and int(rec[0, 2]) == int(lay.sizes.sum()) and _is_identity_move(rec):
            return res._set_blocks(new_layout, self._buf)
        buf = _dest_buffer(new_layout, rec)
        backend.get_lib().copy_blocks(rec, rec_dev, self._buf, buf)
        res._set_blocks(new_layout, buf)
        return res

    def split_legs(self, axes=None, cutoff=0., _view=False):
        """Reshape: split pipes into their incoming legs (reference npc:1707; worker npc:4483 / pyx:1136).
        ``_view``: see :meth:`combine_legs`."""
        if axes is None:
            axes = [i for i, l in enumerate(self.legs) if isinstance(l, LegPipe)]
        elif not isinstance(axes, (list, tuple, np.ndarray)):
            axes = [axes]
        axes = sorted(set(self.get_leg_indices(axes)))
        if len(axes) == 0:
            return self.copy(deep=True)
        for a in axes:
            if not isinstance(self.legs[a], LegPipe):
                raise ValueError('can not split leg {0!r}: not a LegPipe'.format(a))
        res_legs, res_labels = [], []
        for a in range(self.rank):
            if a in axes:
                pipe = self.legs[a]
                res_legs.extend(pipe.legs)
                lab = self._labels[a]
                if lab is not None and lab.startswith('(') and lab.endswith(')'):
                    sub = _split_pipe_label(lab)
                    if len(sub) != pipe.nlegs:
                        sub = [None] * pipe.nlegs
                else:
                    sub = [None] * pipe.nlegs
                res_labels.extend(sub)
            else:
                res_legs.append(self.legs[a])
                res_labels.append(self._labels[a])
        res = Array(res_legs, self.dtype, self.qtotal, res_labels)
        lay = self._layout
        if lay.nblocks == 0:
            return res
        key = ('P', tuple(axes), tuple(self.legs[a].content_key() for a in axes))
        cached = lay.cache.get(key)
        if cached is None:
            new_layout, rec = plan_split(lay, self.legs, axes, res_legs)
            cached = (new_layout, rec, backend.to_device(rec))
            lay.cache[key] = cached
        new_layout, rec, rec_dev = cached
        if _view and new_layout.size == lay.size and int(rec[0, 2]) == int(lay.sizes.sum()) and _is_identity_move(rec):
            return res._set_blocks(new_layout, self._buf)
        buf = _dest_buffer(new_layout, rec)
        backend.get_lib().copy_blocks(rec, rec_dev, self._buf, buf)
        res._set_blocks(new_layout, buf)
        return res

    def as_completely_blocked(self):
        """Wrap non-blocked legs into single-leg pipes (reference npc:1794).

        Returns ``(piped_axes, blocked_self)``."""
        piped = [ax for ax, l in enumerate(self.legs) if not l.is_blocked()]
        if len(piped) == 0:
            return [], self
        res = self.combine_legs([[a] for a in piped], new_axes=piped)
        res._labels = list(self._labels)
        return piped, res

    def gauge_total_charge(self, axis, newqtotal=None, new_qconj=None):
        """Shift the charges of one leg such that ``qtotal`` becomes `newqtotal` (reference npc:1240)."""
        res = self.copy(deep=False)
        ax = self.get_leg_index(axis)
        old = self.legs[ax]
        if isinstance(old, LegPipe):
            old = old.to_LegCharge()
        if new_qconj is None:
            new_qconj = old.qconj
        newqtotal = self.chinfo.make_valid(newqtotal)
        chdiff = newqtotal - self.qtotal
        new_charges = old.charges + old.qconj * chdiff
        if new_qconj != old.qconj:
            new_charges = -new_charges
        leg = LegCharge.from_qind(self.chinfo, old.slices, self.chinfo.make_valid(new_charges), new_qconj)
        res.legs[ax] = leg
        res.qtotal = newqtotal
        return res

    def add_trivial_leg(self, axis=0, label=None, qconj=1):
        """Insert a leg of size 1 with zero charge (reference npc:1187)."""
        if axis < 0:
            axis += self.rank + 1
        leg = LegCharge.from_trivial(1, self.chinfo, qconj)
        res = self.copy(deep=True)
        res.legs.insert(axis, leg)
        res._labels.insert(axis, label)
        res._set_shape()
        lay = self._layout
        qd = np.insert(lay.qdata, axis, 0, axis=1)
        sh = np.insert(lay.shapes, axis, 1, axis=1)
        order = _lexsort_rows(qd) if qd.shape[0] > 1 else np.arange(qd.shape[0])
        if np.any(order != np.arange(len(order))):
            raise NotImplementedError('add_trivial_leg changing the block order')
        res._layout = BlockLayout(qd, sh)
        return res

    def squeeze(self, axes=None):
        """Remove legs of length 1; their charge goes into `qtotal` (reference npc:1817).  Metadata only: the
        packed blocks keep their order and offsets (a unit axis does not change the row-major data)."""
        if axes is None:
            axes = [a for a in range(self.rank) if self.shape[a] == 1]
        else:
            axes = self.get_leg_indices(axes if isinstance(axes, (list, tuple)) else [axes])
        for a in axes:
            if self.shape[a] != 1:
                raise ValueError('Tried to squeeze non-unit leg')
        keep = [a for a in range(self.rank) if a not in axes]
        if len(keep) == 0:
            raise NotImplementedError('squeeze to a scalar: use to_ndarray()')
        res = self.copy(deep=False)
        res.legs = [self.legs[a] for a in keep]
        res._labels = [self._labels[a] for a in keep]
        res._set_shape()
        qtotal = self.qtotal.copy()
        for a in axes:
            qtotal = qtotal - self.legs[a].get_charge(0)
        res.qtotal = self.chinfo.make_valid(qtotal)
        lay = self._layout
        res._layout = BlockLayout(np.ascontiguousarray(lay.qdata[:, keep]), np.ascontiguousarray(lay.shapes[:, keep]))
        return res

    def take_slice(self, indices, axes):
        """``A.take_slice([i, j], [1, 2])`` = ``A[:, i, j, :]`` (reference npc:1037): the legs `axes` are removed,
        their charges at the given indices are subtracted from `qtotal`.  One strided block-copy launch."""
        axes = self.get_leg_indices(list(axes) if isinstance(axes, (list, tuple, np.ndarray)) else [axes])
        indices = np.atleast_1d(np.asarray(indices, dtype=np.intp))
        if len(axes) != len(indices):
            raise ValueError('len(axes) != len(indices)')
        if indices.ndim != 1:
            raise ValueError('indices may only contain ints')
        if len(axes) == 0:
            return self.copy(deep=True)
        pos = np.array([self.legs[a].get_qindex(int(i)) for a, i in zip(axes, indices)], dtype=np.int64)
        keep_axes = [a for a in range(self.rank) if a not in axes]
        qtotal = self.qtotal.copy()
        for a, (qi, _) in zip(axes, pos):
            qtotal = qtotal - self.legs[a].get_charge(int(qi))
        res = Array([self.legs[a] for a in keep_axes], self.dtype, self.chinfo.make_valid(qtotal),
                    [self._labels[a] for a in keep_axes])
        lay = self._layout
        if lay.nblocks == 0:
            return res
        key = ('TS', tuple(axes), pos.tobytes())
        cached = lay.cache.get(key)
        if cached is None:
            new_layout, rec = plan_take_slice(lay, axes, pos[:, 0], pos[:, 1])
            cached = (new_layout, rec, backend.to_device(rec) if new_layout.nblocks else None)
            if len(lay.cache) < 256:
                lay.cache[key] = cached
        new_layout, rec, rec_dev = cached
        if new_layout.nblocks:
            buf = _dest_buffer(new_layout, rec)
            backend.get_lib().copy_blocks(rec, rec_dev, self._buf, buf)
            res._set_blocks(new_layout, buf)
        return res

    def add_leg(self, leg, i, axis=0, label=None):
        """Copy with the new `leg` inserted before `axis`; ``result.take_slice(i, axis)`` is `self`, all other
        entries are zero, `qtotal` grows by the charge of index `i` (reference npc:1130)."""
        if axis < 0:
            axis += self.rank
        legs = list(self.legs)
        legs.insert(axis, leg)
        qi, ri = leg.get_qindex(int(i))
        labels = list(self._labels)
        if label is not None and label in labels:
            raise ValueError('label already exists')
        labels.insert(axis, label)
        res = Array(legs, self.dtype, self.chinfo.make_valid(self.qtotal + leg.get_charge(qi)))
        res._labels = labels
        lay = self._layout
        if lay.nblocks == 0:
            return res
        bs = int(leg.get_block_sizes()[qi])
        key = ('AL', axis, int(qi), int(ri), bs)
        cached = lay.cache.get(key)
        if cached is None:
            new_layout, rec = plan_add_leg(lay, axis, qi, ri, bs)
            cached = (new_layout, rec, backend.to_device(rec))
            if len(lay.cache) < 256:
                lay.cache[key] = cached
        new_layout, rec, rec_dev = cached
        # a unit block needs no zero fill: the copy covers it
        buf = _dest_buffer(new_layout, rec) if bs == 1 else backend.zeros(new_layout.size)
        backend.get_lib().copy_blocks(rec, rec_dev, self._buf, buf)
        return res._set_blocks(new_layout, buf)

    def extend(self, axis, extra):
        """Increase the dimension of `axis` by the blocks of `extra` (LegCharge or int), filled with zeros
        (reference npc:1172).  The stored blocks do not change."""
        res = self.copy(deep=True)
        ax = self.get_leg_index(axis)
        res.legs[ax] = res.legs[ax].extend(extra)
        res._set_shape()
        return res

    def iswapaxes(self, axis1, axis2):
        """Swap two legs in place (reference npc:2090)."""
        a1, a2 = self.get_leg_indices([axis1, axis2])
        perm = list(range(self.rank))
        perm[a1], perm[a2] = a2, a1
        return self.itranspose(perm)

    def is_completely_blocked(self):
        """Reference npc:1368."""
        return all(l.is_blocked() for l in self.legs)

    def isort_qdata(self):
        """The block table of a packed Array is always lex-sorted (reference npc:1431): nothing to do."""
        return self

    def complex_conj(self):
        """Complex conjugate without touching the charges (reference npc:2237); real data: a copy."""
        return self.copy(deep=True)

    def matvec(self, other):
        """``tensordot(self, other, axes=1)`` (reference npc:2364); lets a 2D Array act as a linear operator."""
        return tensordot(self, other, axes=1)

    def __repr__(self):
        return '<npc.Array shape={0!s} labels={1!s} blocks={2:d}>'.format(self.shape, self._labels,
                                                                         self.stored_blocks)

    def sparse_stats(self):
        return '{0:d} of {1:d} entries stored in {2:d} blocks'.format(int(np.sum(self._layout.sizes)), self.size,
                                                                     self.stored_blocks)


def _union_layout(legs, a, b):
    """Union of two block tables on the same legs.

    Returns ``(union_layout, seg_a, seg_b)`` with segment tables (x_off, y_off, len) copying the blocks of
    `a` / `b` into the union buffer."""
    qd = np.concatenate([a.qdata, b.qdata], axis=0)
    order = _lexsort_rows(qd)
    qs = qd[order]
    diffs = charges._row_change_points(qs)
    union = BlockLayout.from_legs(legs, qs[diffs[:-1]], presorted=True)[0]
    target = np.empty(len(qd), dtype=np.int64)
    target[order] = np.repeat(np.arange(len(diffs) - 1), np.diff(diffs))
    ta, tb = target[:a.nblocks], target[a.nblocks:]
    seg_a = np.stack([a.offsets, union.offsets[ta], a.sizes], axis=1) if a.nblocks else np.zeros((0, 3), np.int64)
    seg_b = np.stack([b.offsets, union.offsets[tb], b.sizes], axis=1) if b.nblocks else np.zeros((0, 3), np.int64)
    return union, np.ascontiguousarray(seg_a), np.ascontiguousarray(seg_b)


# ====================================================================== module level functions
def zeros(legcharges, dtype=np.float64, qtotal=None, labels=None):
    """Array without stored blocks (reference npc:3108)."""
    if np.dtype(dtype).kind == 'c':
        return ComplexArray(Array(legcharges, np.float64, qtotal, labels), Array(legcharges, np.float64, qtotal, labels))
    return Array(legcharges, np.float64 if np.dtype(dtype).kind in 'fiub' else dtype, qtotal, labels)


def ones(legcharges, dtype=np.float64, qtotal=None, labels=None):
    """All charge-allowed blocks filled with ones (reference npc:2969)."""
    return Array.from_func(np.ones, legcharges, dtype, qtotal, labels=labels)


def detect_qtotal(flat_array, legcharges, cutoff=None):
    """Total charge of the sector of the largest entry of a dense array (reference npc:3346)."""
    return Array.detect_qtotal(flat_array, legcharges, cutoff)


def concatenate(arrays, axis=0, copy=True):
    """Stack Arrays along `axis` like ``np.concatenate`` (reference npc:3027): the leg is the concatenation of the
    legs (neither sorted nor bunched), every stored block stays a block; labels from the first array.  With a
    :class:`ComplexArray` among `arrays` the real and the imaginary parts are concatenated separately."""
    arrays = list(arrays)
    if any(isinstance(a, ComplexArray) for a in arrays):
        parts = [(a.re, a.im) if isinstance(a, ComplexArray) else (a, a.zeros_like()) for a in arrays]
        return ComplexArray(concatenate([p[0] for p in parts], axis, copy), concatenate([p[1] for p in parts], axis, copy))
    first = arrays[0]
    axis = first.get_leg_index(axis)
    not_axis = [a for a in range(first.rank) if a != axis]
    for a in arrays:
        if a.shape[:axis] != first.shape[:axis] or a.shape[axis + 1:] != first.shape[axis + 1:]:
            raise ValueError('wrong shape to fit ' + repr(a.shape) + ' into ' + repr(first.shape))
        if a.chinfo != first.chinfo:
            raise ValueError('wrong ChargeInfo')
        if np.any(a.qtotal != first.qtotal):
            raise ValueError('wrong qtotal')
        for l in not_axis:
            a.legs[l].test_equal(first.legs[l])
    axis_qconj = first.legs[axis].qconj
    sizes, chs, shifts, shift = [], [], [], 0
    for a in arrays:
        leg = a.legs[axis]
        sizes.extend(leg.get_block_sizes())
        chs.append(leg.charges if leg.qconj == axis_qconj else first.chinfo.make_valid(-leg.charges))
        shifts.append(shift)
        shift += leg.block_number
    new_leg = LegCharge.from_qind(first.chinfo, np.append([0], np.cumsum(sizes)), np.concatenate(chs, axis=0), axis_qconj)
    legs = list(first.legs)
    legs[axis] = new_leg
    res = Array(legs, np.float64, first.qtotal)
    res._labels = list(first._labels)
    key = ('CAT', axis, tuple(a._layout.uid for a in arrays[1:]), tuple(l.content_key() for l in legs))
    cached = first._layout.cache.get(key)
    if cached is None or any(c is not a._layout for c, a in zip(cached[3], arrays)):
        new_layout, recs = plan_concatenate([a._layout for a in arrays], legs, axis, shifts)
        cached = (new_layout, recs, [backend.to_device(r) if len(r) else None for r in recs], [a._layout for a in arrays])
        if len(first._layout.cache) < 256:
            first._layout.cache[key] = cached
    new_layout, recs, recs_dev = cached[:3]
    if new_layout.nblocks == 0:
        return res
    buf = backend.zeros(new_layout.size) if new_layout.has_padding else backend.empty(new_layout.size)
    lib = backend.get_lib()
    for a, rec, rec_dev in zip(arrays, recs, recs_dev):
        if len(rec):
            lib.copy_blocks(rec, rec_dev, a._buf, buf)
    return res._set_blocks(new_layout, buf)


def diag(s, leg, dtype=None, labels=None):
    """2D Array with `s` on the diagonal, legs ``(leg, leg.conj())`` (reference npc:3234); a ComplexArray for complex
    `s`."""
    if np.iscomplexobj(s):
        s = np.asarray(s)
        return ComplexArray(diag(s.real, leg, labels=labels), diag(s.imag, leg, labels=labels))
    s = np.asarray(s, dtype=np.float64)
    scalar = s.ndim == 0
    if not scalar and s.shape != (leg.ind_len,):
        raise ValueError('len(s) does not match leg.ind_len')
    qd = np.arange(leg.block_number, dtype=np.int64)
    blocks = []
    for qi in range(leg.block_number):
        sl = leg.get_slice(qi)
        n = sl.stop - sl.start
        blocks.append(np.eye(n) * float(s) if scalar else np.diag(s[sl]))
    return Array.from_blocks([leg, leg.conj()], np.stack([qd, qd], axis=1), blocks, None, labels)


def eye_like(a, axis=0, labels=None):
    """Identity with legs ``(a.legs[axis], a.legs[axis].conj())`` (reference npc:3211)."""
    return diag(1., a.get_leg(axis), labels=labels)


def _prepare_contraction(a, b, axes):
    """Bring `a`, `b` into standard form: contracted legs last in `a`, first in `b` (reference npc:4666)."""
    if isinstance(axes, (int, np.integer)) and not isinstance(axes, bool):
        n = int(axes)
        axes_a = list(range(a.rank - n, a.rank))
        axes_b = list(range(n))
    else:
        axes_a, axes_b = axes
        if isinstance(axes_a, (str, int, np.integer)):
            axes_a = [axes_a]
        if isinstance(axes_b, (str, int, np.integer)):
            axes_b = [axes_b]
        axes_a = a.get_leg_indices(list(axes_a))
        axes_b = b.get_leg_indices(list(axes_b))
        if len(axes_a) != len(axes_b):
            raise ValueError('different number of axes for a and b')
        n = len(axes_a)
    not_a = [i for i in range(a.rank) if i not in axes_a]
    not_b = [i for i in range(b.rank) if i not in axes_b]
    if a.chinfo != b.chinfo:
        raise ValueError('different ChargeInfo')
    for la, lb in zip(axes_a, axes_b):
        a.legs[la].test_contractible(b.legs[lb])
    a = a.transpose(not_a + axes_a) if not_a + axes_a != list(range(a.rank)) else a
    b = b.transpose(axes_b + not_b) if axes_b + not_b != list(range(b.rank)) else b
    return a, b, n


def tensordot(a, b, axes=2, _out=None, _oz_slices=None):
    """Contract legs of `a` with legs of `b`, like ``np.tensordot`` (reference npc:3612).

    The block products of the whole contraction run as ONE grouped FP64 tensor-core GEMM launch per tile
    shape (worker: reference pyx:1498 / npc:4846).  ``_out`` (internal): device buffer of exactly the result's packed
    size without alignment padding, written instead of a fresh allocation (lets a caller place the result inside a
    larger packed buffer)."""
    if isinstance(a, ComplexArray) or isinstance(b, ComplexArray):
        return _sf.complex_product(_sys.modules[__name__], a, b, lambda x, y: tensordot(x, y, axes))
    a, b, n = _prepare_contraction(a, b, axes)
    cut_a = a.rank - n
    if cut_a == 0 and b.rank == n:
        return inner(a, b, axes='range', do_conj=False)
    res_legs = a.legs[:cut_a] + b.legs[n:]
    res = Array(res_legs, np.float64, a.chinfo.make_valid(a.qtotal + b.qtotal), a._labels[:cut_a] + b._labels[n:]) \
        if _labels_unique(a._labels[:cut_a] + b._labels[n:]) else \
        Array(res_legs, np.float64, a.chinfo.make_valid(a.qtotal + b.qtotal))
    la, lb = a._layout, b._layout
    if la.nblocks == 0 or lb.nblocks == 0:
        return res
    key = (la.uid, lb.uid, n)
    cached = _PLAN_CACHE.get(key)
    if cached is None or cached[0] is not la or cached[1] is not lb:
        lib = backend.get_lib()
        a_rows = np.prod(la.shapes[:, :cut_a], axis=1)
        a_cols = np.prod(la.shapes[:, cut_a:], axis=1)
        b_rows = np.prod(lb.shapes[:, :n], axis=1)
        b_cols = np.prod(lb.shapes[:, n:], axis=1)
        plan = lib.tdot_plan(la.qdata, lb.qdata, n, a_rows, a_cols, la.offsets, b_rows, b_cols, lb.offsets)
        if plan.n_c:
            lay_c = BlockLayout.from_legs(res_legs, plan.c_qdata, presorted=True)[0]
            if lay_c.size != plan.c_size or np.any(lay_c.offsets != plan.c_off):
                raise RuntimeError('internal error: plan / layout offsets disagree')
        else:
            lay_c = None
        if len(_PLAN_CACHE) >= _PLAN_CACHE_MAX:
            _PLAN_CACHE.clear()
        cached = (la, lb, plan, lay_c)
        _PLAN_CACHE[key] = cached
    plan, lay_c = cached[2], cached[3]
    if lay_c is None:
        return res
    if _out is not None:
        if lay_c.has_padding or _out.numel() != lay_c.size:
            raise ValueError('tensordot(_out=...): buffer does not fit the result layout')
        buf = _out
    else:
        buf = backend.zeros(lay_c.size) if lay_c.has_padding else backend.empty(lay_c.size)
    if not (OZAKI['enabled'] and _tensordot_int8(a, b, plan, buf, _oz_slices)):
        plan.run(a._buf, b._buf, buf)
    res._set_blocks(lay_c, buf)
    return res


# Large dense block products can run on the int8 tensor path (wgmma, csrc/ozaki.cu): FP64 operands are cut into signed
# 7-bit digit planes, the slice products are exact integer tensor-core GEMMs, the result is summed in FP64.  `slices`:
# 8 = FP64 rounding level (error ~1e-15 (|A||B|)_ij), 7 (~1e-14) inside the Lanczos matvec (TwoSiteH passes
# `_oz_slices`).  `min_flops` / `min_dim`: below, the DMMA grouped GEMM is as fast and needs no splitting pass.
# Off by default: on the H100 the FP64 tensor cores (DMMA, grouped_gemm_kernel) run the matvec products at 32-41 TFLOP/s,
# the int8 path at 19-22 TFLOP/s FP64-equivalent with 7 digit planes (H100 SXM 80 GB, 700 W, CUDA events, m, n, k from
# 1024 to 4096).
OZAKI = {'enabled': False, 'slices': 8, 'slices_matvec': 7, 'min_flops': 2.e9, 'min_dim': 256, 'calls': 0}


def _oz_split_operand(lib, arr, role, rows, k, off, slices):
    """int8 digit planes of one operand block (rows x k; role 'A': row-major rows x k, role 'B': row-major k x rows);
    cached on Arrays their owner declared constant (``arr._oz_const = True``: the environments of a bond, which every
    Lanczos iteration multiplies again)."""
    cache = None
    if getattr(arr, '_oz_const', False):
        cache = arr.__dict__.setdefault('_oz_cache', {})
        key = (role, slices, int(off), arr._buf.data_ptr())
        hit = cache.get(key)
        if hit is not None:
            return hit
    X = arr._buf[off:]
    sp = lib.ozaki_split(rows, k, X, k, 1, slices) if role == 'A' else lib.ozaki_split(rows, k, X, 1, rows, slices)
    if cache is not None:
        cache[key] = sp
    return sp


def _raw_product(lib, a, b, geom, plan, out, slices=None):
    """one dense block product ``out (m x n) = A (m x k) . B (k x n)`` on raw buffers (internal; replay of recorded
    kernel sequences, see TwoSiteH._dense_recipe_run): `a` / `b` are Arrays (their int8 digit planes are cached when the
    owner declared them constant) or bare device buffers; int8 tensor path when it applies, else the DMMA plan"""
    m, n, k = geom
    if OZAKI['enabled'] and 2. * m * n * k >= OZAKI['min_flops'] and min(m, n, k) >= OZAKI['min_dim'] and \
            hasattr(lib, 'ozaki_mm'):
        s = int(slices or OZAKI['slices'])
        a_s = _oz_split_operand(lib, a, 'A', m, k, 0, s) if isinstance(a, Array) else lib.ozaki_split(m, k, a, k, 1, s)
        b_s = _oz_split_operand(lib, b, 'B', n, k, 0, s) if isinstance(b, Array) else lib.ozaki_split(n, k, b, 1, n, s)
        lib.ozaki_mm(m, n, k, s, a_s, b_s, out, n)
        OZAKI['calls'] += 1
    else:
        plan.run(a._buf if isinstance(a, Array) else a, b._buf if isinstance(b, Array) else b, out)


def _tensordot_int8(a, b, plan, buf, slices=None):
    """run a single large block product of a contraction plan on the int8 tensor path; False if not applicable"""
    if plan.n_c != 1 or plan.n_pairs != 1:
        return False
    lib = backend.get_lib()
    if not hasattr(lib, 'ozaki_mm'):
        return False
    m, n = int(plan.c_rows[0]), int(plan.c_cols[0])
    geom = getattr(plan, '_oz_geom', None)
    if geom is None:
        _, a_off, b_off, kk = plan.pairs()
        geom = plan._oz_geom = (int(a_off[0]), int(b_off[0]), int(kk[0]))
    a_off, b_off, k = geom
    if 2. * m * n * k < OZAKI['min_flops'] or min(m, n, k) < OZAKI['min_dim'] or k > 100000:
        return False
    s = int(slices or OZAKI['slices'])
    a_s = _oz_split_operand(lib, a, 'A', m, k, a_off, s)
    b_s = _oz_split_operand(lib, b, 'B', n, k, b_off, s)
    lib.ozaki_mm(m, n, k, s, a_s, b_s, buf[int(plan.c_off[0]):], n)
    OZAKI['calls'] += 1
    return True


def _is_identity_move(rec):
    """True if the copy records describe ONE contiguous block copied onto the same offsets (a pure relabelling of the
    packed buffer, e.g. combining / splitting legs of an Array without charges)."""
    if len(rec) != 1 or rec[0, 0] != 0 or rec[0, 1] != 0:
        return False
    r = int(rec[0, 3])
    return bool(np.all(rec[0, 10:10 + r] == rec[0, 16:16 + r]))


def _dest_buffer(layout, rec):
    """destination buffer of a block move: zero-filled unless the copy records `rec` cover every element of every
    block and the layout has no alignment padding (then the fill launch is skipped)"""
    if not layout.has_padding and len(rec) and int(rec[:, 2].sum()) == int(layout.sizes.sum()):
        return backend.empty(layout.size)
    return backend.zeros(layout.size)


def _labels_unique(labels):
    seen = [l for l in labels if l is not None]
    return len(seen) == len(set(seen))


def outer(a, b):
    """Outer product (reference npc:3575), via a contraction over zero legs."""
    if isinstance(a, ComplexArray) or isinstance(b, ComplexArray):
        return _sf.complex_product(_sys.modules[__name__], a, b, outer)
    a2, b2, n = _prepare_contraction(a, b, 0)
    res_legs = a.legs + b.legs
    labels = a._labels + b._labels
    res = Array(res_legs, np.float64, a.chinfo.make_valid(a.qtotal + b.qtotal),
                labels if _labels_unique(labels) else None)
    la, lb = a._layout, b._layout
    if la.nblocks == 0 or lb.nblocks == 0:
        return res
    lib = backend.get_lib()
    ones_a = np.ones(la.nblocks, dtype=np.int64)
    ones_b = np.ones(lb.nblocks, dtype=np.int64)
    plan = lib.tdot_plan(la.qdata, lb.qdata, 0, la.sizes, ones_a, la.offsets, ones_b, lb.sizes, lb.offsets)
    lay_c = BlockLayout.from_legs(res_legs, plan.c_qdata, presorted=True)[0]
    buf = backend.zeros(lay_c.size)
    plan.run(a._buf, b._buf, buf)
    res._set_blocks(lay_c, buf)
    return res


def inner(a, b, axes='labels', do_conj=False):
    """Full contraction ``sum a[i,j,..] b[i,j,..]`` (reference npc:3540; worker pyx:1791).

    `axes`: ``'range'`` = leg k of `a` with leg k of `b`; ``'labels'`` (default) = match by label (conjugated
    labels for ``do_conj=False``); or ``(axes_a, axes_b)``.  ``do_conj=True`` conjugates `a` first.
    With a :class:`ComplexArray` operand the result is a ``np.complex128`` (a Python ``complex``), composed of the real
    inner products of the parts."""
    if isinstance(a, list) and isinstance(b, list):
        return sum(inner(w, v, axes=axes, do_conj=do_conj) for w, v in zip(a, b))
    if isinstance(a, ComplexArray) or isinstance(b, ComplexArray):
        a_re, a_im = (a.re, a.im) if isinstance(a, ComplexArray) else (a, None)
        b_re, b_im = (b.re, b.im) if isinstance(b, ComplexArray) else (b, None)
        sgn = 1. if do_conj else -1.          # conj(a) b = (ar br + ai bi) + i (ar bi - ai br)

        def part(x, y):
            return 0. if x is None or y is None else float(inner(x, y, axes=axes, do_conj=do_conj))
        re = part(a_re, b_re) + sgn * part(a_im, b_im)
        im = part(a_re, b_im) - sgn * part(a_im, b_re)
        return np.complex128(complex(re, im))        # (a numpy scalar, like the reference's: np.real(..).item() works)
    if a.rank != b.rank:
        raise ValueError('different rank!')
    if axes != 'range':
        if axes == 'labels':
            a_labels = a.get_leg_labels()
            axes = (a_labels, a_labels) if do_conj else (a_labels, [_conj_label(l) for l in a_labels])
        axes_a, axes_b = axes
        axes_a = a.get_leg_indices(list(axes_a))
        axes_b = b.get_leg_indices(list(axes_b))
        if len(axes_a) != a.rank or len(axes_b) != b.rank:
            raise ValueError('no full contraction. Use tensordot instead!')
        order = np.argsort(axes_b)
        axes_a = [axes_a[i] for i in order]
        if axes_a != list(range(a.rank)):
            a = a.transpose(axes_a)
    if a.chinfo != b.chinfo:
        raise ValueError('different ChargeInfo')
    if do_conj:
        for la_, lb_ in zip(a.legs, b.legs):
            la_.test_equal(lb_)
        if np.any(a.qtotal != b.qtotal):
            return np.float64(0.0)
    else:
        for la_, lb_ in zip(a.legs, b.legs):
            la_.test_contractible(lb_)
        if np.any(a.chinfo.make_valid(a.qtotal + b.qtotal) != 0):
            return np.float64(0.0)
    la, lb = a._layout, b._layout
    if la.nblocks == 0 or lb.nblocks == 0:
        return np.float64(0.0)
    lib = backend.get_lib()
    out = backend.scalar_out()
    if la.same_blocks(lb):
        lib.dot(la.size, a._buf, b._buf, backend.dot_scratch(), out)
        return np.float64(backend.read_scalar(out))
    # intersect the block tables
    qd = np.concatenate([la.qdata, lb.qdata], axis=0)
    order = _lexsort_rows(qd)
    qs = qd[order]
    same = np.nonzero(np.all(qs[1:] == qs[:-1], axis=1))[0]
    if len(same) == 0:
        return np.float64(0.0)
    i1, i2 = order[same], order[same + 1]
    ia = np.where(i1 < la.nblocks, i1, i2)
    ib = np.where(i1 < la.nblocks, i2, i1) - la.nblocks
    seg = np.ascontiguousarray(np.stack([la.offsets[ia], lb.offsets[ib], la.sizes[ia]], axis=1))
    total = 0.0
    # the segment reduction supports up to 2048 partials per launch
    for s0 in range(0, len(seg), 1024):
        part = np.ascontiguousarray(seg[s0:s0 + 1024])
        lib.dot_segments(len(part), backend.to_device(part), int(part[:, 2].max()), a._buf, b._buf,
                         backend.dot_scratch(), out)
        total += backend.read_scalar(out)
    return np.float64(total)


def norm(a, ord=None, convert_to_float=True):
    """Norm of an Array or a plain ndarray (reference npc:3852)."""
    if isinstance(a, Array):
        return a.norm(ord, convert_to_float)
    return float(np.linalg.norm(np.asarray(a).reshape(-1), ord))


def trace(a, leg1=0, leg2=1):
    """Trace of a 2D Array (host reduction over the diagonal blocks; cold path)."""
    if a.rank != 2:
        raise NotImplementedError('trace only for rank 2')
    if isinstance(a, ComplexArray):
        return complex(trace(a.re, leg1, leg2), trace(a.im, leg1, leg2))
    return float(np.trace(a.to_ndarray()))


def _guess_is_orthogonal_basis(G, leg, axis_keep, a_qind):
    """True if the 2D Array `G` is block-wise square (a complete orthonormal basis change of `leg`) and covers
    every sector of `leg` that `a` uses."""
    if G is None or G.rank != 2:
        return False
    try:
        G.legs[axis_keep].test_equal(leg)
    except ValueError:
        return False
    lay = G._layout
    if lay.nblocks == 0 or np.any(lay.shapes[:, 0] != lay.shapes[:, 1]):
        return False
    if G.shape[0] != G.shape[1]:
        return False
    have = set(lay.qdata[:, axis_keep].tolist())
    return all(q in have for q in set(a_qind.tolist()))


# `deflation_tol` used by `svd` when the caller passes none: callers that cannot pass the extension argument (the
# reference's own `svd_theta` running on this engine, tenpy_b200.dropin) set it here
SVD_DEFAULTS = {'deflation_tol': None}
_SVD_LIB_STATE = object()      # internal: "the tolerance is already set in the library"


def svd(a, full_matrices=False, compute_uv=True, cutoff=None, qtotal_LR=[None, None], inner_labels=[None, None],
        inner_qconj=+1, guess=None, deflation_tol=None, n_keep=None):
    """Singular value decomposition ``a = U diag(S) VH`` of a 2D Array (reference npc:3676).

    All charge blocks are decomposed by ONE batched block-Jacobi launch sequence on the device
    (replaces the per-block LAPACK loop of npc:4950).  `S` is block-ordered, descending within a block,
    exactly like the reference's.

    `guess` (extension, optional): ``(U_guess, VH_guess)`` complete orthonormal bases from an earlier SVD of a
    nearby matrix (e.g. the same DMRG bond one sweep ago).  The matrix is rotated into that basis first
    (two extra GEMMs), which makes the Jacobi iteration start almost converged; the result is a full SVD of
    `a` to the usual tolerance whatever the quality of the guess.
    `deflation_tol` (extension, optional): see ``b200_svd_set_deflation_tol`` in include/b200npc.h; ``None``
    keeps the library default (rounding level only, LAPACK-grade factorisation).
    `n_keep` (extension, optional): the caller keeps at most that many singular triplets (``chi_max``); vectors of
    negligible directions beyond it are not completed (they are zero, their `S` is exactly 0).

    A :class:`ComplexArray` `a` is decomposed by the complex block-Jacobi kernel (``b200_block_svd_z``) with the same
    charges, legs and options; `U` and `VH` are then ComplexArrays and `S` is real.  `guess` is not supported for
    complex input (NotImplementedError)."""
    if guess is not None and isinstance(a, ComplexArray):
        raise NotImplementedError('svd: `guess` (warm start) is only implemented for real Arrays')
    if deflation_tol is None:
        deflation_tol = SVD_DEFAULTS['deflation_tol']        # module-wide default (None: rounding level only)
    if deflation_tol is not None and deflation_tol is not _SVD_LIB_STATE:
        lib0 = backend.get_lib()
        old_tol = lib0.svd_set_deflation_tol(deflation_tol)
        try:
            return svd(a, full_matrices, compute_uv, cutoff, qtotal_LR, inner_labels, inner_qconj, guess, _SVD_LIB_STATE,
                       n_keep)
        finally:
            lib0.svd_set_deflation_tol(old_tol)
    if guess is not None and compute_uv and cutoff is None and not full_matrices and a.rank == 2:
        Ug, VHg = guess
        chinfo = a.chinfo
        qtotal_L, qtotal_R = qtotal_LR
        if qtotal_L is None and qtotal_R is None:
            qtotal_R = a.qtotal
        if qtotal_L is None:
            qtotal_L = chinfo.make_valid(a.qtotal - qtotal_R)
        elif qtotal_R is None:
            qtotal_R = chinfo.make_valid(a.qtotal - qtotal_L)
        qtotal_L, qtotal_R = chinfo.make_valid(qtotal_L), chinfo.make_valid(qtotal_R)
        if a.legs[0].is_blocked() and a.legs[1].is_blocked() and a._layout.nblocks:
            if _guess_is_orthogonal_basis(Ug, a.legs[0], 0, a._layout.qdata[:, 0]):
                a2 = tensordot(Ug.conj(), a, axes=[0, 0])
                a2.iset_leg_labels([None, a._labels[1]])
                U2, S, VH = svd(a2, qtotal_LR=[chinfo.make_valid(qtotal_L - Ug.qtotal), qtotal_R],
                                inner_labels=inner_labels, inner_qconj=inner_qconj, n_keep=n_keep)
                U = tensordot(Ug, U2, axes=[1, 0])
                U.iset_leg_labels([a._labels[0], inner_labels[0]])
                svd_stats['guess_used'] = svd_stats.get('guess_used', 0) + 1
                return U, S, VH
            if _guess_is_orthogonal_basis(VHg, a.legs[1], 1, a._layout.qdata[:, 1]):
                a2 = tensordot(a, VHg.conj(), axes=[1, 1])
                a2.iset_leg_labels([a._labels[0], None])
                U, S, VH2 = svd(a2, qtotal_LR=[qtotal_L, chinfo.make_valid(qtotal_R - VHg.qtotal)],
                                inner_labels=inner_labels, inner_qconj=inner_qconj, n_keep=n_keep)
                VH = tensordot(VH2, VHg, axes=[1, 0])
                VH.iset_leg_labels([inner_labels[1], a._labels[1]])
                svd_stats['guess_used'] = svd_stats.get('guess_used', 0) + 1
                return U, S, VH
    if a.rank != 2:
        raise ValueError('SVD is only defined for a 2D matrix. Use LegPipes!')
    if full_matrices:
        raise NotImplementedError('full_matrices=True is not needed on the DMRG path')
    labL, labR = inner_labels
    a_labels = a._labels
    piped_axes, a = a.as_completely_blocked()
    chinfo = a.chinfo
    qtotal_L, qtotal_R = qtotal_LR
    if qtotal_L is None and qtotal_R is None:
        qtotal_R = a.qtotal
    if qtotal_L is None:
        qtotal_L = chinfo.make_valid(a.qtotal - qtotal_R)
    elif qtotal_R is None:
        qtotal_R = chinfo.make_valid(a.qtotal - qtotal_L)
    elif np.any(a.qtotal != chinfo.make_valid(np.asarray(qtotal_L) + np.asarray(qtotal_R))):
        raise ValueError('The entries of `qtotal_LR` have to add up to ``a.qtotal``!')
    qtotal_L = chinfo.make_valid(qtotal_L)
    qtotal_R = chinfo.make_valid(qtotal_R)
    cplx = isinstance(a, ComplexArray)
    if cplx:
        lay, bufA_re, bufA_im = _complex_planes(a)
    else:
        lay = a._layout
    if lay.nblocks == 0:
        raise RuntimeError('SVD found no singular values')
    m = lay.shapes[:, 0]
    n = lay.shapes[:, 1]
    k = np.minimum(m, n)
    s_off = np.concatenate(([0], np.cumsum(k)))
    # new inner leg (reference npc:5017-5026)
    qi_L, qi_R = lay.qdata[:, 0], lay.qdata[:, 1]
    new_charges = chinfo.make_valid((qtotal_R - a.legs[1].get_charge(qi_R)) * inner_qconj)
    new_leg_R = LegCharge.from_qind(chinfo, s_off, new_charges, inner_qconj)
    new_leg_L = new_leg_R.conj()
    qi_C = np.arange(lay.nblocks, dtype=np.int64)
    U = Array([a.legs[0], new_leg_L], np.float64, qtotal_L)
    VH = Array([new_leg_R, a.legs[1]], np.float64, qtotal_R)
    lay_U, perm_U = BlockLayout.from_legs(U.legs, np.stack([qi_L, qi_C], axis=1))
    lay_V, perm_V = BlockLayout.from_legs(VH.legs, np.stack([qi_C, qi_R], axis=1))
    u_off = np.empty(lay.nblocks, dtype=np.int64)
    v_off = np.empty(lay.nblocks, dtype=np.int64)
    u_off[perm_U] = lay_U.offsets
    v_off[perm_V] = lay_V.offsets
    lib = backend.get_lib()
    bufU = backend.zeros(lay_U.size)
    bufV = backend.zeros(lay_V.size)
    bufS = backend.empty(int(s_off[-1]))
    if cplx:
        bufU_im = backend.zeros(lay_U.size)
        bufV_im = backend.zeros(lay_V.size)
        info, nact, transp = lib.block_svd_z(m, n, lay.offsets, u_off, s_off[:-1], v_off, bufA_re, bufA_im, bufU, bufU_im,
                                             bufS, bufV, bufV_im)
    else:
        info, nact, transp = lib.block_svd(m, n, lay.offsets, u_off, s_off[:-1], v_off, a._buf, bufU, bufS, bufV)
    svd_stats['calls'] += 1
    svd_stats['jacobi_sweeps'].append(int(np.max(info)))
    if np.any(nact < k):
        # numerically rank-deficient blocks: the kernel left the vectors of the negligible directions on one side zero;
        # complete them to an orthonormal basis (LAPACK returns a complete basis, reference npc:4950).  Real blocks: GEMM-only
        # Newton-Schulz, which can fail on an ill-conditioned start; complex blocks: the complex QR kernel, which cannot
        if cplx:
            fill, fill_U, fill_V = _fill_null_vectors_z, (bufU, bufU_im), (bufV, bufV_im)
        else:
            fill, fill_U, fill_V = _fill_null_vectors, bufU, bufV
        S_h = backend.to_host(bufS).copy()
        try:
            for i in np.nonzero(nact < k)[0]:
                # the caller keeps at most `n_keep` vectors in total (svd_theta: chi_max): no need to complete more
                k_fill = int(k[i]) if n_keep is None else min(int(k[i]), max(int(n_keep), int(nact[i])))
                n_fill = k_fill - int(nact[i])
                if n_fill > 0:
                    fill(lib, int(m[i]), int(n[i]), int(k[i]), int(nact[i]), n_fill, bool(transp[i]), fill_U, int(u_off[i]),
                         fill_V, int(v_off[i]))
                # singular values of the negligible directions: tiny but positive for the completed vectors (so that a
                # truncation prefers them), exactly zero for the ones left without a vector
                lo, hi = int(s_off[i]) + int(nact[i]), int(s_off[i]) + int(k[i])
                S_h[lo:lo + n_fill] = np.maximum(S_h[lo:lo + n_fill], _completion_floor(S_h[int(s_off[i]):lo]))
                S_h[lo + n_fill:hi] = 0.
        except _CompletionFailed:
            # real blocks only: decompose once more without deflation, every direction iterated to convergence
            svd_stats['completion_fallbacks'] = svd_stats.get('completion_fallbacks', 0) + 1
            old = lib.svd_set_deflation(False)
            try:
                bufU.zero_()
                bufV.zero_()
                info, nact, transp = lib.block_svd(m, n, lay.offsets, u_off, s_off[:-1], v_off, a._buf, bufU, bufS, bufV)
            finally:
                lib.svd_set_deflation(old)
        else:
            svd_stats['completions'] = svd_stats.get('completions', 0) + 1
            bufS = backend.to_device(S_h)
    S = backend.to_host(bufS)
    if np.any(np.isnan(S)):
        raise ValueError('NaN in S')
    if not compute_uv:
        if cutoff is not None:
            S = S[S > cutoff]
        return S
    U._set_blocks(lay_U, bufU)
    VH._set_blocks(lay_V, bufV)
    if cplx:
        U_im = Array(U.legs, np.float64, U.qtotal)._set_blocks(lay_U, bufU_im)
        VH_im = Array(VH.legs, np.float64, VH.qtotal)._set_blocks(lay_V, bufV_im)
        U, VH = ComplexArray(U, U_im), ComplexArray(VH, VH_im)
    if cutoff is not None:
        keep = S > cutoff
        if not np.any(keep):
            raise RuntimeError('SVD found no singular values')
        S = S[keep]
        U.iproject(keep, 1)
        VH.iproject(keep, 0)
    if 0 in piped_axes:
        U = U.split_legs(0)
    if 1 in piped_axes:
        VH = VH.split_legs(1)
    U.iset_leg_labels([a_labels[0], labL])
    VH.iset_leg_labels([labR, a_labels[1]])
    return U, S, VH


class _CompletionFailed(Exception):
    pass


def _completion_floor(S_genuine):
    """lower bound of the singular value of a completed (negligible) direction of a block whose genuine singular values
    are `S_genuine` (all > 0: they exceed the deflation threshold): 1e-99, but at most eps times the smallest genuine one
    (and never below the smallest positive double, nor above the smallest genuine one), so that a truncation keeps the
    genuine directions of a block first at any scale of the block, U S VH stays A to eps, and the bound stays > 0."""
    if not len(S_genuine):
        return 1.e-99
    smin = float(np.min(S_genuine))
    return min(1.e-99, smin, max(smin * np.finfo(np.float64).eps, 5e-324))


_SMALL_DEV_CACHE = {}     # small constant device arrays (copy records, index lists, the scalar 1.) by content


def _dev_const(key, make):
    """device copy of a small constant host array, made once (every host->device copy of a record is a driver call)"""
    ent = _SMALL_DEV_CACHE.get(key)
    if ent is None or ent[0] is not backend.get_lib():
        if len(_SMALL_DEV_CACHE) > 4096:
            _SMALL_DEV_CACHE.clear()
        host = make()
        ent = _SMALL_DEV_CACHE[key] = (backend.get_lib(), host, backend.to_device(host))
    return ent[1], ent[2]


def _strided_copy(lib, src, soff, dst, doff, shape, sstride, dstride):
    def make():
        rec = np.zeros((1, 22), dtype=np.int64)
        r = len(shape)
        rec[0, 0], rec[0, 1], rec[0, 2], rec[0, 3] = soff, doff, int(np.prod(shape)), r
        rec[0, 4:10] = 1
        rec[0, 4:4 + r] = shape
        rec[0, 10:10 + r] = sstride
        rec[0, 16:16 + r] = dstride
        return rec
    rec, rec_dev = _dev_const(('copy', soff, doff, tuple(shape), tuple(sstride), tuple(dstride)), make)
    lib.copy_blocks(rec, rec_dev, src, dst)


def _gemm(lib, mm, nn, kk, A, B, C):
    lib.grouped_gemm([mm], [nn], [0], [0, 1], [kk], [0], [0], A, B, C)


def _null_space_completion(lib, V, r, p, kf):
    """`kf` orthonormal rows (device buffer, kf x p row-major) orthogonal to the `r` orthonormal rows of `V`.

    Start from projected unit vectors ``X0 = E_sel - C^T V`` with ``C = V[:, sel]`` for the `kf` coordinates of
    smallest leverage (so that ``X0 X0^T = 1 - C^T C`` is well conditioned), then orthonormalise with
    Newton-Schulz iterations ``X <- (1 - D/2) X``, ``D = X X^T - 1`` -- GEMMs only (grouped FP64 tensor-core
    kernel).  Left multiplications keep the rows inside the orthogonal complement of `V`."""
    ones = _dev_const('one', lambda: np.ones(1))[1]
    X = backend.zeros(kf * p)
    if r > 0:
        lev = backend.empty(p)
        lib.col_sqnorms(r, p, p, V, lev)
        sel = np.sort(np.argsort(backend.to_host(lev), kind='stable')[:kf]).astype(np.int64)
        C = backend.empty(r * kf)
        rec = np.array([[0, 0, r, kf, 1, p, 0]], dtype=np.int64)
        lib.take_blocks(rec, backend.to_device(rec), backend.to_device(sel), V, C)
        CT = backend.empty(kf * r)
        _strided_copy(lib, C, 0, CT, 0, [kf, r], [1, kf], [r, 1])
        _gemm(lib, kf, p, r, CT, V, X)
        lib.scal(kf * p, -1., X)
    else:
        sel = np.arange(kf, dtype=np.int64)
    seg = np.stack([np.zeros(kf, np.int64), np.arange(kf, dtype=np.int64) * p + sel, np.ones(kf, np.int64)], axis=1)
    for s0 in range(0, kf, 32768):
        part = np.ascontiguousarray(seg[s0:s0 + 32768])
        lib.axpy_segments(len(part), backend.to_device(part), 1, 1., ones, X)
    if r == 0:
        return X
    dseg_dev = [_dev_const(('diag', kf, s0), lambda s0=s0: np.ascontiguousarray(np.stack(
        [np.zeros(kf, np.int64), np.arange(kf, dtype=np.int64) * (kf + 1), np.ones(kf, np.int64)], axis=1)[s0:s0 + 32768]))[1]
        for s0 in range(0, kf, 32768)]
    XT = backend.empty(kf * p)
    G = backend.empty(kf * kf)
    DX = backend.empty(kf * p)
    out = backend.scalar_out()
    for it in range(60):
        _strided_copy(lib, X, 0, XT, 0, [p, kf], [1, p], [kf, 1])
        _gemm(lib, kf, kf, p, X, XT, G)
        for dsd in dseg_dev:
            lib.axpy_segments(dsd.shape[0], dsd, 1, -1., ones, G)
        lib.dot(kf * kf, G, G, backend.dot_scratch(), out)
        err = float(np.sqrt(backend.read_scalar(out)))
        if not np.isfinite(err) or (it == 0 and err > np.sqrt(kf) * (1. - 1e-7)):
            raise _CompletionFailed('ill-conditioned start')
        if err < 1e-13 * max(1., np.sqrt(kf)):
            return X
        _gemm(lib, kf, p, kf, G, X, DX)
        lib.axpy(kf * p, -0.5, DX, X)
    raise _CompletionFailed('Newton-Schulz did not converge')


def _fill_null_vectors(lib, m, n, k, r, kf, transposed, bufU, u_off, bufV, v_off):
    """fill `kf` of the zero vectors left by the deflating SVD kernel for block (m x n), see b200_block_svd_f64"""
    if not transposed:           # rows r..k-1 of VT (k x n) are missing; the first r rows are orthonormal
        V = bufV[v_off:v_off + max(r, 1) * n]
        X = _null_space_completion(lib, V, r, n, kf)
        bufV[v_off + r * n:v_off + (r + kf) * n].copy_(X[:kf * n])
    else:                        # columns r..k-1 of U (m x k) are missing
        V = backend.empty(max(r, 1) * m)
        if r > 0:
            _strided_copy(lib, bufU, u_off, V, 0, [r, m], [1, k], [m, 1])
        X = _null_space_completion(lib, V, r, m, kf)
        _strided_copy(lib, X, 0, bufU, u_off + r, [kf, m], [m, 1], [1, k])


def _fill_null_vectors_z(lib, m, n, k, r, kf, transposed, bufU, u_off, bufV, v_off):
    """complex counterpart of :func:`_fill_null_vectors` (`bufU`, `bufV` = (real, imaginary) planes): the `r` orthonormal
    vectors `v_i` (length `p`) of the accumulated side, followed by the `kf` unit vectors of smallest leverage, are the
    columns of ``M`` (p x (r + kf)); the Householder QR kernel gives ``M = Q R`` with orthonormal columns, the first `r`
    spanning the `v_i`, so columns ``r .. r+kf-1`` of `Q` are orthonormal and orthogonal to them.  Unlike the
    Newton-Schulz completion this cannot fail: the reflectors are unitary whatever the conditioning of `M`."""
    p = m if transposed else n
    c = r + kf
    rows = [backend.empty(max(r, 1) * p) for _ in range(2)]     # the r vectors as rows (r x p), both planes
    if r > 0:
        for part, buf in enumerate(bufU if transposed else bufV):
            if transposed:          # columns 0..r-1 of U (m x k)
                _strided_copy(lib, buf, u_off, rows[part], 0, [r, m], [1, k], [m, 1])
            else:                   # rows 0..r-1 of VT (k x n)
                rows[part][:r * n].copy_(buf[v_off:v_off + r * n])
        lev = backend.empty(p)
        lev_im = backend.empty(p)
        lib.col_sqnorms(r, p, p, rows[0], lev)
        lib.col_sqnorms(r, p, p, rows[1], lev_im)
        sel = np.sort(np.argsort(backend.to_host(lev) + backend.to_host(lev_im), kind='stable')[:kf]).astype(np.int64)
    else:
        sel = np.arange(kf, dtype=np.int64)
    M = [backend.zeros(p * c) for _ in range(2)]
    if r > 0:
        for part in range(2):
            _strided_copy(lib, rows[part], 0, M[part], 0, [r, p], [p, 1], [1, c])
    ones = _dev_const('one', lambda: np.ones(1))[1]
    seg = np.ascontiguousarray(np.stack([np.zeros(kf, np.int64), sel * c + r + np.arange(kf, dtype=np.int64),
                                         np.ones(kf, np.int64)], axis=1))
    lib.axpy_segments(len(seg), backend.to_device(seg), 1, 1., ones, M[0])
    Q = [backend.empty(p * c) for _ in range(2)]
    R = [backend.empty(c * c) for _ in range(2)]
    lib.block_qr_z([p], [c], [0], [0], [0], M[0], M[1], Q[0], Q[1], R[0], R[1])
    for part in range(2):
        if transposed:              # columns r.. of U <- columns r.. of Q
            _strided_copy(lib, Q[part], r, bufU[part], u_off + r, [p, kf], [c, 1], [k, 1])
        else:                       # rows r.. of VT <- columns r.. of Q
            _strided_copy(lib, Q[part], r, bufV[part], v_off + r * n, [kf, p], [1, c], [p, 1])


def _complex_planes(a):
    """``(layout, buf_re, buf_im)``: the two parts of the ComplexArray `a` on ONE block table.  Each part drops its own
    zero blocks, so their tables can differ; a block missing in one part is a zero block there."""
    lr, li = a.re._layout, a.im._layout
    if lr.same_blocks(li):
        return lr, a.re._buf, a.im._buf
    union, seg_re, seg_im = _union_layout(a.legs, lr, li)
    lib = backend.get_lib()
    bufs = []
    for seg, part in ((seg_re, a.re), (seg_im, a.im)):
        buf = backend.zeros(union.size)
        if len(seg):
            lib.axpy_segments(len(seg), backend.to_device(seg), int(seg[:, 2].max()), 1.0, part._buf, buf)
        bufs.append(buf)
    return union, bufs[0], bufs[1]


qr_stats = {'calls': 0, 'columns': 0, 'replaced': 0}   # diagnostics of the Gram-Schmidt QR
# real blocks of up to QR_HOUSEHOLDER_MAX rows and columns: b200_block_qr_f64, one CTA per block, one launch for all of
# them; larger real blocks: Gram-Schmidt on the GEMM / BLAS-1 kernels (one host round trip per column)
QR_HOUSEHOLDER_MAX = 384


_SQ_SAFE = (2.**-900, 2.**900)     # squared norms in this range leave the Gram-Schmidt sums far from over- and underflow


def _rescale_column(lib, m, v, sq, scratch, out):
    """Norm of the column `v` (device, length `m`, squared norm `sq`) after scaling it in place by powers of two
    (exact) until its squared norm lies in `_SQ_SAFE`; a column already in range is left untouched, a zero column stays
    zero.  Gram-Schmidt is invariant under column scaling (``A D = Q (R D)``), and R is formed from the unscaled A."""
    for _ in range(4):
        if _SQ_SAFE[0] <= sq <= _SQ_SAFE[1] or not sq == sq:
            break
        if sq == 0.:
            e = 600
        elif sq == np.inf:
            e = -600
        else:
            e = -(int(np.frexp(sq)[1]) // 2)
        lib.scal(m, 2.**e, v)
        lib.dot(m, v, v, scratch, out)
        sq = float(backend.read_scalar(out))
    return float(np.sqrt(max(sq, 0.)))


def _block_qr_cgs2(lib, m, n, A, Q, R):
    """``A (m x n) = Q (m x k) R (k x n)``, ``k = min(m, n)``, on device buffers (row-major views): classical
    Gram-Schmidt with re-orthogonalisation ("twice is enough"), column by column, built from the existing kernels --
    two skinny GEMMs per pass (projection on the previous vectors), one dot + one scal per column -- and
    ``R = Q^T A`` by one GEMM with the strictly lower triangle dropped.  A column that is linearly dependent on the
    previous ones (norm after projection below ``64 eps`` of its original norm) is replaced by an orthonormalised unit
    vector, so that `Q` stays an isometry (LAPACK's Householder QR returns an orthonormal completion there, too).

    Cost model: one host round trip per column (the norm).  This is a functional stand-in on the cold paths
    (`MPS.canonical_form`); a batched Householder kernel is round-2 work (DESIGN.md section 8)."""
    k = min(m, n)
    out = backend.scalar_out()
    scratch = backend.dot_scratch()
    T = backend.empty(n * m)                                   # T = A^T: row j = column j of A (contiguous)
    _strided_copy(lib, A, 0, T, 0, [n, m], [1, n], [m, 1])
    cn = backend.empty(n)
    lib.col_sqnorms(m, n, n, A, cn)
    col_sq = backend.to_host(cn)
    Qt = backend.zeros(k * m)
    w = backend.empty(max(k, 1))
    tmp = backend.empty(m)
    ones = backend.to_device(np.ones(1))
    next_unit = 0
    for j in range(k):
        v = T[j * m:(j + 1) * m].clone()
        col_norm = _rescale_column(lib, m, v, float(col_sq[j]), scratch, out)
        replaced = False
        while True:
            for _ in range(2):
                if j > 0:
                    _gemm(lib, j, 1, m, Qt[:j * m], v, w[:j])          # w = Q_{<j}^T v
                    _gemm(lib, 1, m, j, w[:j], Qt[:j * m], tmp)        # tmp = w^T Q_{<j}^T
                    lib.axpy(m, -1., tmp, v)
            lib.dot(m, v, v, scratch, out)
            nrm = float(np.sqrt(max(backend.read_scalar(out), 0.)))
            ref = 1. if replaced else col_norm
            if nrm > 64 * np.finfo(np.float64).eps * ref and nrm > 0.:
                break
            # dependent column: continue with a unit vector (the next one not yet tried)
            if next_unit >= m:
                raise RuntimeError('QR: could not complete the isometry')
            v = backend.zeros(m)
            seg = np.array([[0, next_unit, 1]], dtype=np.int64)
            lib.axpy_segments(1, backend.to_device(seg), 1, 1., ones, v)
            next_unit += 1
            replaced = True
            qr_stats['replaced'] += 1
        lib.scal(m, 1. / nrm, v)
        Qt[j * m:(j + 1) * m].copy_(v)
    qr_stats['columns'] += k
    _strided_copy(lib, Qt, 0, Q, 0, [m, k], [1, m], [k, 1])
    Rfull = backend.empty(k * n)
    _gemm(lib, k, n, m, Qt, A, Rfull)
    rec = np.zeros((k, 22), dtype=np.int64)                        # row i of R: entries i .. n-1
    i = np.arange(k, dtype=np.int64)
    rec[:, 0] = rec[:, 1] = i * n + i
    rec[:, 2] = n - i
    rec[:, 3] = 1
    rec[:, 4:10] = 1
    rec[:, 4] = n - i
    rec[:, 10] = rec[:, 16] = 1
    lib.copy_blocks(rec, backend.to_device(rec), Rfull, R)


def qr(a, mode='reduced', inner_labels=[None, None], cutoff=None, pos_diag_R=False, qtotal_Q=None, inner_qconj=+1):
    """Q-R decomposition ``a == tensordot(Q, R, axes=1)`` per charge block (reference npc:4139): `Q` an isometry with
    legs ``(a.legs[0], inner.conj())``, `R` upper triangular with legs ``(inner, a.legs[1])``.

    Only ``mode='reduced'`` and ``cutoff=None``.  The diagonal of `R` is non-negative by construction (Householder kernel
    ``b200_block_qr_f64`` for blocks of up to `QR_HOUSEHOLDER_MAX` rows and columns, Gram-Schmidt :func:`_block_qr_cgs2`
    above), i.e. the result is the unique decomposition the reference returns for ``pos_diag_R=True`` (for full-rank
    blocks).  A :class:`ComplexArray` `a` goes through the complex Householder kernel
    (``b200_block_qr_z``, every block size); `Q` and `R` are then ComplexArrays, the diagonal of `R` real and >= 0."""
    if a.rank != 2:
        raise ValueError('expect a matrix!')
    if mode != 'reduced':
        raise NotImplementedError("qr: only mode='reduced'")
    if cutoff is not None:
        raise NotImplementedError('qr with cutoff (pivoted QR discarding dependent columns)')
    a_labels = a._labels
    label_Q, label_R = inner_labels
    piped_axes, a = a.as_completely_blocked()
    chinfo = a.chinfo
    cplx = isinstance(a, ComplexArray)
    if cplx:
        lay, bufA_re, bufA_im = _complex_planes(a)
    else:
        lay = a._layout
    a_leg0 = a.legs[0]
    m, n = lay.shapes[:, 0], lay.shapes[:, 1]
    k = np.minimum(m, n)
    # the new inner leg = the row sectors that have a block, truncated to k (reference npc:4190-4215)
    mask = np.zeros(a_leg0.ind_len, dtype=np.bool_)
    for q1, kk in zip(lay.qdata[:, 0], k):
        i0 = int(a_leg0.slices[q1])
        mask[i0:i0 + int(kk)] = True
    inner_leg = a_leg0.to_LegCharge() if isinstance(a_leg0, LegPipe) else a_leg0.copy()
    map_qind, _, inner_leg = inner_leg.project(mask)
    charges_in = inner_leg.charges
    if qtotal_Q is not None:
        qtotal_Q = chinfo.make_valid(qtotal_Q)
        charges_in = chinfo.make_valid(charges_in - inner_leg.qconj * qtotal_Q)
    qc = inner_leg.qconj
    if qc != inner_qconj:
        charges_in = chinfo.make_valid(-charges_in)
        qc = inner_qconj
    inner_leg = LegCharge.from_qind(chinfo, inner_leg.slices, charges_in, qc)
    Q = Array([a_leg0, inner_leg.conj()], np.float64, qtotal_Q)
    R = Array([inner_leg, a.legs[1]], np.float64, chinfo.make_valid(a.qtotal - Q.qtotal))
    if lay.nblocks:
        qi_C = map_qind[lay.qdata[:, 0]].astype(np.int64)
        lay_Q, perm_Q = BlockLayout.from_legs(Q.legs, np.stack([lay.qdata[:, 0], qi_C], axis=1))
        lay_R, perm_R = BlockLayout.from_legs(R.legs, np.stack([qi_C, lay.qdata[:, 1]], axis=1))
        q_off = np.empty(lay.nblocks, dtype=np.int64)
        r_off = np.empty(lay.nblocks, dtype=np.int64)
        q_off[perm_Q] = lay_Q.offsets
        r_off[perm_R] = lay_R.offsets
        bufQ = backend.zeros(lay_Q.size)
        bufR = backend.zeros(lay_R.size)
        lib = backend.get_lib()
        if cplx:         # complex: the Householder kernel for every block size
            Q_im, R_im = Array(Q.legs, np.float64, Q.qtotal), Array(R.legs, np.float64, R.qtotal)
            bufQ_im = backend.zeros(lay_Q.size)
            bufR_im = backend.zeros(lay_R.size)
            lib.block_qr_z(m, n, lay.offsets, q_off, r_off, bufA_re, bufA_im, bufQ, bufQ_im, bufR, bufR_im)
            Q_im._set_blocks(lay_Q, bufQ_im)
            R_im._set_blocks(lay_R, bufR_im)
        else:
            small = np.maximum(m, n) <= QR_HOUSEHOLDER_MAX
            if np.any(small):
                lib.block_qr(m[small], n[small], lay.offsets[small], q_off[small], r_off[small], a._buf, bufQ, bufR)
            for b in np.nonzero(~small)[0]:
                mb, nb, kb = int(m[b]), int(n[b]), int(k[b])
                ao = int(lay.offsets[b])
                _block_qr_cgs2(lib, mb, nb, a._buf[ao:ao + mb * nb], bufQ[int(q_off[b]):int(q_off[b]) + mb * kb],
                               bufR[int(r_off[b]):int(r_off[b]) + kb * nb])
        Q._set_blocks(lay_Q, bufQ)
        R._set_blocks(lay_R, bufR)
        qr_stats['calls'] += 1
    elif cplx:
        Q_im, R_im = Array(Q.legs, np.float64, Q.qtotal), Array(R.legs, np.float64, R.qtotal)
    if cplx:
        Q, R = ComplexArray(Q, Q_im), ComplexArray(R, R_im)
    if 0 in piped_axes:
        Q = Q.split_legs(0)
    if 1 in piped_axes:
        R = R.split_legs(-1)
    Q.iset_leg_labels([a_labels[0], label_Q])
    R.iset_leg_labels([label_R, a_labels[1]])
    return Q, R


def pinv(a, cutoff=1.e-15):
    """Moore-Penrose pseudo-inverse via svd (reference npc:3821)."""
    labels = a.get_leg_labels()
    U, S, VH = svd(a, cutoff=cutoff)
    VH.iscale_axis(1. / S, 0)
    res = tensordot(VH.conj().itranspose(), U.conj().itranspose(), axes=1)
    return res.iset_leg_labels([labels[1], labels[0]]) if _labels_unique([labels[1], labels[0]]) else res


def eigvalsh(a, UPLO='L', sort=None):
    """Eigenvalues of a hermitian 2D Array (reference npc:3972)."""
    return eigh(a, UPLO, sort)[0]


def _hermitian_defect(a):
    """``(|a - a^H|_F^2, |a|_F^2)`` of the square ComplexArray `a`: four dot products on the device, one read back"""
    d = a - a.conj().itranspose()
    lib = backend.get_lib()
    out = backend.zeros(4)
    for j, part in enumerate((d.re, d.im, a.re, a.im)):
        lay = part._layout
        if lay.nblocks:
            lib.dot(lay.size, part._buf, part._buf, backend.dot_scratch(), out[j:j + 1])
    r = backend.to_host(out)
    return float(r[0] + r[1]), float(r[2] + r[3])


def eigh(a, UPLO='L', sort=None):
    """Eigen-decomposition of a hermitian 2D Array with contractible legs (reference npc:3899 / :5041).

    Returns ``(W, V)``: eigenvalues (1D host array, ordered like the first leg; within a block ascending or
    as requested by `sort`) and the unitary `V` with legs ``(a.legs[0], a.legs[0].conj() as LegCharge)``.
    Missing diagonal blocks give eigenvalue 0 with unit vectors, exactly like the reference.
    A :class:`ComplexArray` `a` must be Hermitian to ``|a - a^H|_F <= 1e-8 |a|_F`` (else NotImplementedError: only
    Hermitian eigenproblems are provided); it goes through the complex block-Jacobi kernel (``b200_block_eigh_z``), `W`
    is real and `V` a ComplexArray."""
    cplx = isinstance(a, ComplexArray)
    if a.rank != 2 or a.shape[0] != a.shape[1]:
        raise ValueError('expect a square matrix!')
    a.legs[0].test_contractible(a.legs[1])
    if np.any(a.qtotal != a.chinfo.make_valid()):
        raise ValueError('Non-trivial qtotal -> Nilpotent. Not diagonizable!?')
    if cplx:
        defect2, norm2 = _hermitian_defect(a)
        if not defect2 <= 1e-16 * norm2:
            raise NotImplementedError('eigh: the ComplexArray is not complex Hermitian (|A - A^H|_F = {0:.3g} |A|_F); '
                                      'only Hermitian eigenproblems are provided'.format(
                                          np.sqrt(defect2 / norm2) if norm2 > 0. else np.inf))
    a_label0 = a._labels[0]
    piped_axes, a = a.as_completely_blocked()
    leg = a.legs[0]
    if cplx:
        lay, bufA, bufA_im = _complex_planes(a)
    else:
        lay, bufA = a._layout, a._buf
    if np.any(lay.qdata[:, 0] != lay.qdata[:, 1]):
        raise ValueError('off-diagonal blocks in a completely blocked matrix with zero charge?')
    resw = np.zeros(a.shape[0], dtype=np.float64)
    # V: identity blocks for all sectors, overwritten for the stored ones
    nbk = leg.block_number
    sizes = leg.get_block_sizes().astype(np.int64)
    leg2 = a.legs[1].to_LegCharge() if isinstance(a.legs[1], LegPipe) else a.legs[1]
    V = Array([leg, leg2], np.float64, None)
    qd = np.arange(nbk, dtype=np.int64)
    lay_V = BlockLayout.from_legs(V.legs, np.stack([qd, qd], axis=1), presorted=True)[0]
    stored = lay.qdata[:, 0]
    missing = np.setdiff1d(qd, stored)
    if len(missing):
        host = np.zeros(lay_V.size, dtype=np.float64)
        for qi in missing:
            nq = int(sizes[qi])
            o = int(lay_V.offsets[qi])
            host[o:o + nq * nq] = np.eye(nq).reshape(-1)
        bufV = backend.to_device(host)
    else:
        bufV = backend.zeros(lay_V.size)
    planes = [bufV]
    if cplx:
        planes.append(backend.zeros(lay_V.size))
    if lay.nblocks:
        lib = backend.get_lib()
        nn = sizes[stored]
        w_off = np.concatenate(([0], np.cumsum(nn)))
        bufW = backend.empty(int(w_off[-1]))
        if cplx:
            lib.block_eigh_z(nn, lay.offsets, w_off[:-1], lay_V.offsets[stored], bufA, bufA_im, bufW, bufV, planes[1])
        else:
            lib.block_eigh(nn, lay.offsets, w_off[:-1], lay_V.offsets[stored], bufA, bufW, bufV)
        w = backend.to_host(bufW)
        recs, pool, at = [], [], 0
        for j, qi in enumerate(stored):
            rw = w[w_off[j]:w_off[j + 1]]
            if sort is not None and sort != '<':
                # order inside the block as requested (reference tools/misc.py argsort): permute the eigenvalues
                # on the host and the columns of V with one take launch (per plane)
                key = {'m<': np.abs(rw), 'm>': -np.abs(rw), '>': -rw}.get(sort)
                if key is None:
                    raise ValueError('unknown sort option ' + repr(sort))
                perm = np.argsort(key, kind='stable')
                if np.any(perm != np.arange(len(perm))):
                    nq = len(rw)
                    recs.append([int(lay_V.offsets[qi]), int(lay_V.offsets[qi]), nq, nq, 1, nq, at])
                    pool.append(perm.astype(np.int64))
                    at += nq
                    rw = rw[perm]
            resw[leg.get_slice(qi)] = rw
        if recs:
            rec = np.array(recs, dtype=np.int64)
            rec_dev, pool_dev = backend.to_device(rec), backend.to_device(np.concatenate(pool))
            for buf in planes:
                src = buf.clone()
                lib.take_blocks(rec, rec_dev, pool_dev, src, buf)
    V._set_blocks(lay_V, bufV)
    if cplx:
        V_im = Array(V.legs, np.float64, None)
        V_im._set_blocks(lay_V, planes[1])
        V = ComplexArray(V, V_im)
    if len(piped_axes) > 0:
        V = V.split_legs(0)
    V.iset_leg_labels([a_label0, 'eig'] if a_label0 != 'eig' else [None, 'eig'])
    return resw, V


def to_iterable_arrays(array_list):
    """Flatten nested lists of Arrays (reference npc:2996).  An Array (ComplexArray included), a string (an operator name,
    as in ``MPS.expectation_value('Sz')``) or any other non-iterable is one entry."""
    if isinstance(array_list, (Array, str)) or not np.iterable(array_list):
        return [array_list]
    return list(itertools.chain.from_iterable(to_iterable_arrays(a) for a in array_list))


def concatenate_qdata(*a):  # pragma: no cover - placeholder for API completeness
    raise NotImplementedError


# ---- the rest of the reference's surface (cold paths: model / MPO / site construction, indexing, complex tensors) ----------
import sys as _sys

from . import _surface as _sf
from .charges import DipolarChargeInfo
from ._surface import (QCUTOFF, grid_outer, grid_concat, detect_grid_outer_legcharge, detect_legcharge, eig, eigvals,
                       speigs, expm, lq, polar, orthogonal_columns)

Array.__getitem__ = _sf.array_getitem
Array.__setitem__ = _sf.array_setitem
Array.__iter__ = _sf.array_iter
Array.__eq__ = _sf.array_eq
Array.__hash__ = object.__hash__
Array.permute = _sf.array_permute
Array.sort_legcharge = _sf.array_sort_legcharge
Array.unary_blockwise = _sf.array_unary_blockwise
Array.iunary_blockwise = _sf.array_iunary_blockwise
Array.binary_blockwise = _sf.array_binary_blockwise
Array.ipurge_zeros = _sf.array_ipurge_zeros
Array.from_func_square = classmethod(_sf.array_from_func_square)
Array.add_charge = _sf.array_add_charge
Array.drop_charge = _sf.array_drop_charge
Array.change_charge = _sf.array_change_charge
Array.shift_charges = _sf.array_shift_charges
Array.shift_charges_horizontal = _sf.array_shift_charges_horizontal
ComplexArray = _sf._finish_complex(_sys.modules[__name__])

__all__ += ['DipolarChargeInfo', 'QCUTOFF', 'ComplexArray', 'grid_outer', 'grid_concat', 'detect_grid_outer_legcharge',
            'detect_legcharge', 'eig', 'eigvals', 'speigs', 'expm', 'lq', 'polar', 'orthogonal_columns']
