"""Complex tensors: :class:`ComplexArray` gives complex128 tensors as a pair of real device Arrays (same legs, planar
storage); elementwise operations, contractions and inner products are composed of the real kernels.  It carries the
reference's `Site` operators (``Sy`` & co.), real-time evolution and ground states of complex Hamiltonians: ``npc.svd``,
``npc.qr`` and ``npc.eigh`` of a ComplexArray run the complex block kernels (``b200_block_svd_z``, ``b200_block_qr_z``,
``b200_block_eigh_z``) on the (real, imaginary) planes of its blocks (:func:`_planes`).

Imported at the end of ``np_conserved.py``, where :class:`Array` already exists.
"""
import numpy as np

from .. import backend
from .np_conserved import Array, norm, _union_layout


class _WriteThroughBlock(np.ndarray):
    """host copy of one stored block; item assignments are written through to the device: to the block of a real Array
    (which refuses complex values), or to the blocks of both parts of a ComplexArray (see :meth:`Array.get_block`)"""
    _targets = None       # ((device buffer, offset, size), ...): the real part, then the imaginary part

    def __setitem__(self, key, value):
        if self.dtype.kind != 'c' and np.iscomplexobj(value):
            raise TypeError('a block of a real Array can not hold complex values: assign to the blocks of a '
                            'ComplexArray (.re / .im)')
        np.ndarray.__setitem__(self, key, value)
        if self._targets is not None:
            for (buf, o, s), part in zip(self._targets, (np.real, np.imag)):
                buf[o:o + s].copy_(backend.to_device(np.ascontiguousarray(part(self), dtype=np.float64).reshape(-1)))

    def __array_finalize__(self, obj):
        self._targets = None          # views / results of arithmetic are plain host data


class ComplexArray(Array):
    """complex128 tensor = two real device Arrays ``re``, ``im`` on the same legs (see the module doc string); a
    subclass of :class:`Array`, so the ``isinstance`` checks of the reference hold."""

    def __init__(self, re, im):
        self.re, self.im = re, im
        self.legs = list(re.legs)
        self._labels = list(re._labels)
        self.rank, self.shape = re.rank, re.shape
        self.dtype = np.dtype(np.complex128)
        self.chinfo, self.qtotal = re.chinfo, re.qtotal
        self._qdata_sorted = True

    # ---- construction / conversion
    @classmethod
    def from_ndarray(cls, data_flat, legcharges, dtype=None, qtotal=None, cutoff=None, labels=None,
                     raise_wrong_sector=True, warn_wrong_sector=True):
        data_flat = np.asarray(data_flat, dtype=np.complex128)
        legcharges = list(legcharges)
        if qtotal is None:
            qtotal = Array.detect_qtotal(data_flat, legcharges, cutoff)
        kw = dict(qtotal=qtotal, cutoff=cutoff, labels=labels, raise_wrong_sector=raise_wrong_sector,
                  warn_wrong_sector=warn_wrong_sector)
        return cls(Array.from_ndarray(np.ascontiguousarray(data_flat.real), legcharges, **kw),
                   Array.from_ndarray(np.ascontiguousarray(data_flat.imag), legcharges, **kw))

    @classmethod
    def from_blocks(cls, legcharges, qdata, blocks, qtotal=None, labels=None):
        blocks = [np.asarray(b, dtype=np.complex128) for b in blocks]
        return cls(Array.from_blocks(legcharges, qdata, [np.ascontiguousarray(b.real) for b in blocks], qtotal, labels),
                   Array.from_blocks(legcharges, qdata, [np.ascontiguousarray(b.imag) for b in blocks], qtotal, labels))

    def to_ndarray(self):
        return self.re.to_ndarray() + 1.j * self.im.to_ndarray()

    def copy(self, deep=True):
        return ComplexArray(self.re.copy(deep), self.im.copy(deep))

    def astype(self, dtype, copy=True):
        if np.dtype(dtype).kind == 'c':
            return self.copy(deep=True) if copy else self
        if norm(self.im) > 0.:
            import warnings
            warnings.warn('discarding the imaginary part', stacklevel=2)
        return self.re.copy(deep=True)

    @property
    def stored_blocks(self):
        return max(self.re.stored_blocks, self.im.stored_blocks)

    @property
    def size(self):
        return self.re.size

    @property
    def _layout(self):
        raise NotImplementedError('a ComplexArray has no single packed layout (real and imaginary part separately)')

    def get_blocks_host(self):
        raise NotImplementedError('block access of a ComplexArray: use .re / .im')

    def get_block(self, qindices, insert=False, raise_incomp_q=False):
        """the block as a complex host array, or None; stored in both parts (``insert=True`` stores zero blocks
        first), item assignments are written through to both device buffers (``block[:] = values`` as in the
        reference's ``full_diag_effH``, dmrg.py:1209)"""
        a = self.re.get_block(qindices, insert, raise_incomp_q)
        b = self.im.get_block(qindices, insert, raise_incomp_q)
        if a is None and b is None:
            return None
        if a is None or b is None:
            return (0. if a is None else np.asarray(a)) + 1.j * (0. if b is None else np.asarray(b))
        blk = (np.asarray(a) + 1.j * np.asarray(b)).view(_WriteThroughBlock)
        blk._targets = a._targets + b._targets
        return blk

    def test_sanity(self):
        self.re.test_sanity()
        self.im.test_sanity()

    def zeros_like(self):
        return ComplexArray(self.re.zeros_like(), self.im.zeros_like())

    def __repr__(self):
        return '<npc.ComplexArray shape={0!s} labels={1!s}>'.format(self.shape, self._labels)

    def __getstate__(self):
        return {'re': self.re, 'im': self.im}

    def __setstate__(self, state):
        self.__init__(state['re'], state['im'])

    # ---- labels: keep both parts and the wrapper in step
    def _sync(self):
        self.legs = list(self.re.legs)
        self._labels = list(self.re._labels)
        self.rank, self.shape = self.re.rank, self.re.shape
        self.qtotal = self.re.qtotal
        return self

    # ---- arithmetic
    def iconj(self, complex_conj=True):
        self.re.iconj()
        self.im.iconj()
        if complex_conj:
            self.im.iscale_prefactor(-1.)
        return self._sync()

    def conj(self, complex_conj=True):
        return self.copy(deep=True).iconj(complex_conj)

    def complex_conj(self):
        return ComplexArray(self.re.copy(deep=True), self.im * -1.)

    def iscale_prefactor(self, prefactor):
        z = complex(prefactor)
        if z.imag == 0.:
            self.re.iscale_prefactor(z.real)
            self.im.iscale_prefactor(z.real)
        else:
            re = self.re * z.real - self.im * z.imag
            im = self.re * z.imag + self.im * z.real
            self.re, self.im = re, im
        return self

    def iadd_prefactor_other(self, prefactor, other):
        z = complex(prefactor)
        o_re, o_im = (other.re, other.im) if isinstance(other, ComplexArray) else (other, None)
        if z.real != 0.:
            self.re.iadd_prefactor_other(z.real, o_re)
            if o_im is not None:
                self.im.iadd_prefactor_other(z.real, o_im)
        if z.imag != 0.:
            self.im.iadd_prefactor_other(z.imag, o_re)
            if o_im is not None:
                self.re.iadd_prefactor_other(-z.imag, o_im)
        return self

    def __mul__(self, other):
        if np.isscalar(other):
            return self.copy(deep=True).iscale_prefactor(other)
        return NotImplemented

    __rmul__ = __mul__

    def __imul__(self, other):
        return self.iscale_prefactor(other) if np.isscalar(other) else NotImplemented

    def __truediv__(self, other):
        return self.__mul__(1. / other) if np.isscalar(other) else NotImplemented

    def __itruediv__(self, other):
        return self.iscale_prefactor(1. / other) if np.isscalar(other) else NotImplemented

    def __neg__(self):
        return self.__mul__(-1.)

    def __add__(self, other):
        return self.copy(deep=True).iadd_prefactor_other(1., other) if isinstance(other, Array) else NotImplemented

    __radd__ = __add__

    def __iadd__(self, other):
        return self.iadd_prefactor_other(1., other) if isinstance(other, Array) else NotImplemented

    def __sub__(self, other):
        return self.copy(deep=True).iadd_prefactor_other(-1., other) if isinstance(other, Array) else NotImplemented

    def __rsub__(self, other):
        return (self * -1.).iadd_prefactor_other(1., other) if isinstance(other, Array) else NotImplemented

    def __isub__(self, other):
        return self.iadd_prefactor_other(-1., other) if isinstance(other, Array) else NotImplemented

    def norm(self, ord=None, convert_to_float=True):
        return float(np.hypot(self.re.norm(ord), self.im.norm(ord)))

    def scale_axis(self, s, axis=-1):
        return self.copy(deep=True).iscale_axis(s, axis)

    def iscale_axis(self, s, axis=-1):
        """``(re + i im) (sr + i si)`` slice by slice along `axis`"""
        s = np.asarray(s)
        if np.iscomplexobj(s) and np.any(s.imag != 0.):
            sr, si = np.ascontiguousarray(s.real), np.ascontiguousarray(s.imag)
            re = self.re.scale_axis(sr, axis) - self.im.scale_axis(si, axis)
            self.im = self.re.scale_axis(si, axis) + self.im.scale_axis(sr, axis)
            self.re = re
        else:
            self.re.iscale_axis(s.real, axis)
            self.im.iscale_axis(s.real, axis)
        return self._sync()

    def iproject(self, mask, axes):
        self.im.iproject(mask, axes)
        out = self.re.iproject(mask, axes)
        self._sync()
        return out


# methods that act on both parts in the same way and return `self` / a new tensor
def _inplace(name):
    def f(self, *args, **kwargs):
        getattr(self.re, name)(*args, **kwargs)
        getattr(self.im, name)(*args, **kwargs)
        return self._sync()
    f.__name__ = name
    return f


def _outofplace(name):
    def f(self, *args, **kwargs):
        return ComplexArray(getattr(self.re, name)(*args, **kwargs), getattr(self.im, name)(*args, **kwargs))
    f.__name__ = name
    return f


for _name in ('iset_leg_labels', 'ireplace_label', 'ireplace_labels', 'idrop_labels', 'itranspose', 'iswapaxes',
              'isort_qdata'):
    setattr(ComplexArray, _name, _inplace(_name))
for _name in ('transpose', 'replace_label', 'replace_labels', 'combine_legs', 'split_legs', 'take_slice', 'add_leg',
              'extend', 'add_trivial_leg', 'squeeze', 'gauge_total_charge'):
    setattr(ComplexArray, _name, _outofplace(_name))

# pickles name the class by its public place, np_conserved.ComplexArray, not by the module that defines it: so pickles
# written by earlier versions load, and new ones do not depend on where the class is defined
ComplexArray.__module__ = Array.__module__


def _planes(a):
    """``(layout, planes)``: the block table of `a` and its device buffers on it, ``(buf,)`` for an Array and
    ``(buf_re, buf_im)`` for a ComplexArray.  Each part of a ComplexArray drops its own zero blocks, so their tables can
    differ; then both are copied to the union of the tables, where a block missing in one part is a zero block."""
    if not isinstance(a, ComplexArray):
        return a._layout, (a._buf,)
    lr, li = a.re._layout, a.im._layout
    if lr.same_blocks(li):
        return lr, (a.re._buf, a.im._buf)
    union, seg_re, seg_im = _union_layout(a.legs, lr, li)
    lib = backend.get_lib()
    bufs = []
    for seg, part in ((seg_re, a.re), (seg_im, a.im)):
        buf = backend.zeros(union.size)
        if len(seg):
            lib.axpy_segments(len(seg), backend.to_device(seg), int(seg[:, 2].max()), 1.0, part._buf, buf)
        bufs.append(buf)
    return union, tuple(bufs)


def _from_planes(legs, qtotal, layout, planes, labels=None):
    """the Array (one plane) or ComplexArray (real and imaginary plane) on `legs` with the blocks of `layout` in the
    device buffers `planes`; ``layout=None``: without blocks"""
    parts = [Array(legs, np.float64, qtotal, labels) for _ in planes]
    if layout is not None:
        for part, buf in zip(parts, planes):
            part._set_blocks(layout, buf)
    return parts[0] if len(parts) == 1 else ComplexArray(*parts)


def complex_product(a, b, prod):
    """the bilinear product ``prod`` (tensordot, outer) with at least one ComplexArray operand, from the real products
    of the parts"""
    a_re, a_im = (a.re, a.im) if isinstance(a, ComplexArray) else (a, None)
    b_re, b_im = (b.re, b.im) if isinstance(b, ComplexArray) else (b, None)
    re = prod(a_re, b_re)
    if a_im is not None and b_im is not None:
        re = re - prod(a_im, b_im)
    im = None
    if b_im is not None:
        im = prod(a_re, b_im)
    if a_im is not None:
        t = prod(a_im, b_re)
        im = t if im is None else im + t
    if not isinstance(re, Array):          # full contraction: scalars
        return complex(re, im)
    return ComplexArray(re, im)
