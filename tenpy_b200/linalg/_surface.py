"""The part of the `np_conserved` surface (reference ``npc.__all__``, np_conserved.py:106-141, and `Array` methods) that
the reference's networks / models / algorithms use OUTSIDE the two-site DMRG hot path: building sites, MPOs and initial
states, indexing, sorting of leg charges, element-wise functions, small dense factorizations.  These are cold paths
(model construction, measurements); they are implemented on top of the hot-path primitives of
:mod:`tenpy_b200.linalg.np_conserved` (block moves, tensordot, eigh on the device) and, where the reference itself works
element by element on the host (``from_ndarray``, ``__setitem__`` of a few numbers), by one host round trip of the small
tensor involved.  Imported at the end of ``np_conserved.py``, which attaches the methods to :class:`Array`.  Complex
tensors (`ComplexArray`) are in :mod:`tenpy_b200.linalg._complex`.
"""
import numpy as np

from . import charges as _ch
from .charges import LegCharge, LegPipe, QTYPE

__all__ = ['QCUTOFF', 'grid_outer', 'grid_concat', 'detect_grid_outer_legcharge', 'detect_legcharge', 'eig',
           'eigvals', 'speigs', 'expm', 'lq', 'polar', 'orthogonal_columns']

QCUTOFF = np.finfo(np.float64).eps * 10.   # reference np_conserved.py:146


def _npc():
    from . import np_conserved
    return np_conserved


# ------------------------------------------------------------------------------------------------ indexing
def _normalize_inds(arr, inds):
    """per-axis index objects (None = take everything) from the argument of ``a[...]`` (reference npc:3041)"""
    if not isinstance(inds, tuple):
        inds = (inds,)
    n_ell = sum(1 for i in inds if i is Ellipsis)
    if n_ell > 1:
        raise IndexError("an index can only have a single ellipsis ('...')")
    if n_ell == 1:
        e = inds.index(Ellipsis)
        fill = arr.rank - (len(inds) - 1)
        inds = inds[:e] + (slice(None),) * fill + inds[e + 1:]
    if len(inds) > arr.rank:
        raise IndexError('too many indices for Array')
    inds = inds + (slice(None),) * (arr.rank - len(inds))
    return inds


def _as_mask(ind, n):
    """slice / bool mask / sorted index array -> (mask, permutation or None)"""
    if isinstance(ind, slice):
        idx = np.arange(n)[ind]
    else:
        ind = np.asarray(ind)
        idx = np.nonzero(ind)[0] if ind.dtype == np.bool_ else ind.astype(np.intp)
        idx = np.where(idx < 0, idx + n, idx)
    mask = np.zeros(n, dtype=np.bool_)
    mask[idx] = True
    if len(np.unique(idx)) != len(idx):
        raise NotImplementedError('repeated indices in Array.__getitem__')
    order = None if np.all(np.diff(idx) > 0) else np.argsort(np.argsort(idx))
    return mask, order


def array_getitem(self, inds):
    """``a[inds]``: integers remove a leg (`take_slice`), slices / masks / index arrays project it (`iproject`), as the
    reference's ``Array.__getitem__`` (np_conserved.py:920).  All-integer indices return the scalar entry."""
    inds = _normalize_inds(self, inds)
    int_axes = [a for a, i in enumerate(inds) if isinstance(i, (int, np.integer))]
    if len(int_axes) == self.rank:
        pos = [int(i) + (self.shape[a] if i < 0 else 0) for a, i in enumerate(inds)]
        qi = [leg.get_qindex(p) for leg, p in zip(self.legs, pos)]
        blk = self.get_block([q for q, _ in qi])
        return self.dtype.type(0) if blk is None else blk[tuple(r for _, r in qi)]
    res = self
    proj_axes, masks, perms = [], [], []
    for a, i in enumerate(inds):
        if a in int_axes or (isinstance(i, slice) and i == slice(None)):
            continue
        mask, order = _as_mask(i, self.shape[a])
        proj_axes.append(a)
        masks.append(mask)
        perms.append(order)
    if proj_axes:
        res = res.copy(deep=True)
        res.iproject(masks, proj_axes)
        for a, order in zip(proj_axes, perms):
            if order is not None:      # the projection keeps the indices sorted: entry i is the order[i]-th of them
                res = res.permute(order, a)
    if int_axes:
        res = res.take_slice([int(inds[a]) + (self.shape[a] if inds[a] < 0 else 0) for a in int_axes], int_axes)
    return res


def array_setitem(self, inds, other):
    """``a[inds] = other`` (reference npc:971): `other` an Array (or scalar) with the legs the indexing leaves; entries
    that would violate the charge rule raise ValueError.  A host round trip of `self` -- used by the reference when it
    assembles small tensors (MPO matrices in `grid_outer`, initial environments)."""
    npc = _npc()
    inds = _normalize_inds(self, inds)
    dense = self.to_ndarray()
    val = other.to_ndarray() if isinstance(other, npc.Array) else other
    if np.iscomplexobj(val) and not np.iscomplexobj(dense):
        raise TypeError('a real Array can not hold complex values: assign to a ComplexArray (a.astype(complex))')
    np_inds = tuple(int(i) if isinstance(i, (int, np.integer)) else (i if isinstance(i, slice) else np.asarray(i))
                    for i in inds)
    dense[np_inds] = val
    new = type(self).from_ndarray(dense, self.legs, dtype=dense.dtype, qtotal=self.qtotal, cutoff=0., labels=self._labels)
    _adopt(self, new)


def _adopt(self, new):
    """make `self` the tensor `new` (same legs)"""
    if type(new) is not type(self):
        self.__class__ = type(new)
    self.__dict__.update(new.__dict__)


def array_iter(self):
    """iterate over the first leg (reference npc:897)"""
    for i in range(self.shape[0]):
        yield self[i]


def array_eq(self, other, eps=1.e-14):
    """same legs, same total charge and ``norm(self - other) < eps`` (reference npc:2466)"""
    npc = _npc()
    if self is other:
        return True
    if not isinstance(other, npc.Array):
        return NotImplemented
    if other.chinfo != self.chinfo:
        raise ValueError('other array has different charges!')
    other = other._match_labels_of(self)
    if self.rank != other.rank or self.shape != other.shape or np.any(self.qtotal != other.qtotal):
        return False
    return bool(npc.norm(self - other) < eps)


# ------------------------------------------------------------------------------------------------ leg reordering
def array_permute(self, perm, axis):
    """permute the indices of one leg: ``res[..., i, ...] = self[..., perm[i], ...]`` (reference npc:1822); the new leg
    has one charge sector per index run of equal charge (not bunched further)"""
    ax = self.get_leg_index(axis)
    perm = np.asarray(perm, dtype=np.intp)
    leg = self.legs[ax]
    if isinstance(leg, LegPipe):
        leg = leg.to_LegCharge()
    qflat = leg.to_qflat()[perm]
    new_leg = LegCharge.from_qflat(self.chinfo, qflat, leg.qconj)
    dense = np.take(self.to_ndarray(), perm, axis=ax)
    legs = list(self.legs)
    legs[ax] = new_leg
    return type(self).from_ndarray(dense, legs, dtype=dense.dtype, qtotal=self.qtotal, cutoff=0., labels=self._labels)


def array_sort_legcharge(self, sort=True, bunch=True):
    """sort (and bunch) the charge sectors of the legs (reference npc:1735).  Returns ``(perm_flat per leg, result)``."""
    if sort is True or sort is False:
        sort = [sort] * self.rank
    if bunch is True or bunch is False:
        bunch = [bunch] * self.rank
    perms = [None] * self.rank
    res = self
    for ax in range(self.rank):
        s, b = sort[ax], bunch[ax]
        leg = res.legs[ax]
        if isinstance(s, (list, np.ndarray)) and not isinstance(s, (bool, np.bool_)):
            raise NotImplementedError('sort_legcharge with an explicit permutation')
        if s and not leg.is_sorted():
            if isinstance(leg, LegPipe):
                leg = leg.to_LegCharge()
            perm_qind, _ = leg.sort(bunch=False)
            pflat = leg.perm_flat_from_perm_qind(perm_qind)
            perms[ax] = pflat
            res = res.permute(pflat, ax)
            leg = res.legs[ax]
        if b and not leg.is_bunched():
            if isinstance(leg, LegPipe):
                leg = leg.to_LegCharge()
            _, new_leg = leg.bunch()
            dense = res.to_ndarray()
            legs = list(res.legs)
            legs[ax] = new_leg
            res = type(res).from_ndarray(dense, legs, dtype=dense.dtype, qtotal=res.qtotal, cutoff=0., labels=res._labels)
    if res is self:
        res = self.copy(deep=True)
    return tuple(perms), res


# ------------------------------------------------------------------------------------------------ element-wise
def array_unary_blockwise(self, func, *args, **kwargs):
    """``func(block, *args, **kwargs)`` on every stored block (reference npc:2184); `func` is a numpy function, so the
    blocks make one host round trip (measurement code: ``np.abs``, ``np.real`` ...)"""
    return self.copy(deep=True).iunary_blockwise(func, *args, **kwargs)


def array_iunary_blockwise(self, func, *args, **kwargs):
    npc = _npc()
    blocks = [np.asarray(func(b, *args, **kwargs)) for b in self.get_blocks_host()]
    new = type(self).from_blocks(self.legs, self._layout.qdata, blocks, self.qtotal, self._labels) if blocks else \
        npc.Array(self.legs, np.float64, self.qtotal, self._labels)
    _adopt(self, new)
    return self


def array_binary_blockwise(self, other, func, *args, **kwargs):
    """``func(self_block, other_block)`` on the union of the stored blocks (reference npc:2303)"""
    npc = _npc()
    a, b = self.to_ndarray(), other._match_labels_of(self).to_ndarray()
    return type(self).from_ndarray(func(a, b, *args, **kwargs), self.legs, qtotal=self.qtotal, cutoff=0., labels=self._labels)


def array_ipurge_zeros(self, cutoff=QCUTOFF, norm_order=None):
    """drop stored blocks whose norm is below `cutoff` (reference npc:1901)"""
    blocks = self.get_blocks_host()
    keep = [i for i, b in enumerate(blocks) if np.linalg.norm(b.ravel(), ord=norm_order) > cutoff]
    if len(keep) < len(blocks):
        new = type(self).from_blocks(self.legs, self._layout.qdata[keep], [blocks[i] for i in keep], self.qtotal, self._labels)
        _adopt(self, new)
    return self


def array_from_func_square(cls, func, leg, dtype=None, func_args=(), func_kwargs={}, labels=None):
    """square block-diagonal Array on ``[leg, leg.conj()]`` with ``func((n, n))`` in every diagonal block (reference
    npc:712; used for random unitaries)"""
    blocks, qd = [], []
    for qi, n in enumerate(leg.get_block_sizes()):
        blocks.append(np.asarray(func((int(n), int(n)), *func_args, **func_kwargs)))
        qd.append([qi, qi])
    res = cls.from_blocks([leg, leg.conj()], np.array(qd, dtype=np.int64), blocks, None, labels)
    return res


# ------------------------------------------------------------------------------------------------ charges of the legs
def _rebuild_with_legs(self, legs, qtotal):
    dense = self.to_ndarray()
    return type(self).from_ndarray(dense, legs, dtype=dense.dtype, qtotal=qtotal, cutoff=0., labels=self._labels)


def array_add_charge(self, add_legs, chinfo=None, qtotal=None):
    """add charges: the new ChargeInfo is the sum of the old and the one of `add_legs` (reference npc:1203)"""
    if chinfo is None:
        chinfo = _ch.ChargeInfo.add([self.chinfo, add_legs[0].chinfo])
    legs = [LegCharge.from_add_charge([leg.to_LegCharge() if isinstance(leg, LegPipe) else leg, leg2], chinfo)
            for leg, leg2 in zip(self.legs, add_legs)]
    q2 = np.zeros(add_legs[0].chinfo.qnumber, QTYPE) if qtotal is None else np.asarray(qtotal, QTYPE)
    return _rebuild_with_legs(self, legs, np.concatenate([self.qtotal, q2]))


def array_drop_charge(self, charge=None, chinfo=None):
    """remove a charge (reference npc:1232)"""
    if chinfo is None:
        chinfo = _ch.ChargeInfo.drop(self.chinfo, charge)
    legs = [LegCharge.from_drop_charge(leg.to_LegCharge() if isinstance(leg, LegPipe) else leg, charge, chinfo)
            for leg in self.legs]
    if charge is None:
        qtotal = None
    else:
        idx = self.chinfo.names.index(charge) if isinstance(charge, str) else charge
        qtotal = np.delete(self.qtotal, idx)
    return _rebuild_with_legs(self, legs, qtotal)


def array_change_charge(self, charge, new_qmod, new_name='', chinfo=None):
    """change the modulus of a charge (reference npc:1260)"""
    if chinfo is None:
        chinfo = _ch.ChargeInfo.change(self.chinfo, charge, new_qmod, new_name)
    legs = [LegCharge.from_change_charge(leg.to_LegCharge() if isinstance(leg, LegPipe) else leg, charge, new_qmod,
                                         new_name, chinfo) for leg in self.legs]
    return _rebuild_with_legs(self, legs, chinfo.make_valid(self.qtotal))


def array_shift_charges(self, dx, inplace=False):
    """charges after a lattice translation (reference npc:1488): the identity, the engine has no dipole charges"""
    return self


def array_shift_charges_horizontal(self, dx_0, inplace=False):
    return self


# ------------------------------------------------------------------------------------------------ grids
def _grid_entries(grid):
    """(shape, [(index tuple, Array)]) of the non-None entries of an array-like of Arrays"""
    npc = _npc()
    g = np.empty(np.shape(np.asarray([[None]], dtype=object)), dtype=object)   # placeholder, replaced below

    def shape_of(x):
        if isinstance(x, (list, tuple)):
            return (len(x),) + (shape_of(x[0]) if len(x) else ())
        if isinstance(x, np.ndarray) and x.dtype == object:
            return x.shape
        return ()
    shp = shape_of(grid)
    g = np.empty(shp, dtype=object)
    for idx in np.ndindex(*shp):
        x = grid
        for i in idx:
            x = x[i]
        g[idx] = x
    entries = [(idx, g[idx]) for idx in np.ndindex(*shp) if g[idx] is not None]
    for _, e in entries:
        if not isinstance(e, npc.Array):
            raise ValueError('grid entries have to be Arrays or None')
    if not entries:
        raise ValueError('No non-trivial entries in grid')
    return shp, entries


def grid_outer(grid, grid_legs, qtotal=None, grid_labels=None):
    """An array-like `grid` of Arrays (``None`` = zero) as ONE Array with the grid axes in front: ``res[idx] == grid[idx]``
    (reference npc:3206; builds the MPO matrices in ``MPO.from_grids``, networks/mpo.py)."""
    npc = _npc()
    shp, entries = _grid_entries(grid)
    if len(shp) != len(grid_legs):
        raise ValueError('wrong number of grid_legs')
    if shp != tuple(l.ind_len for l in grid_legs):
        raise ValueError('grid shape incompatible with grid_legs')
    idx0, first = entries[0]
    chinfo = first.chinfo
    is_complex = any(e.dtype.kind == 'c' for _, e in entries)
    legs = list(grid_legs) + list(first.legs)
    labels = list(grid_labels) if grid_labels is not None else [None] * len(shp)
    inner_labels = list(first._labels)
    for _, e in entries:
        if e._labels != inner_labels:
            inner_labels = [None] * first.rank
    if qtotal is None:
        q = np.array(first.qtotal, dtype=QTYPE)
        for i, leg in zip(idx0, grid_legs):
            q = q + leg.get_charge(leg.get_qindex(i)[0]) * leg.qconj
        qtotal = chinfo.make_valid(q)
    dense = np.zeros(shp + first.shape, dtype=np.complex128 if is_complex else np.float64)
    for idx, e in entries:
        if e.shape != first.shape:
            raise ValueError('grid entries of different shape')
        dense[idx] = e.to_ndarray()
    return npc.Array.from_ndarray(dense, legs, dtype=dense.dtype, qtotal=qtotal, cutoff=0., labels=labels + inner_labels)


def detect_grid_outer_legcharge(grid, grid_legs, qtotal=None, qconj=1, bunch=False):
    """the one missing (``None``) entry of `grid_legs` such that :func:`grid_outer` gives total charge `qtotal`
    (reference npc:3292); the new leg is neither sorted nor bunched"""
    shp, entries = _grid_entries(grid)
    if len(shp) != len(grid_legs):
        raise ValueError('wrong number of grid_legs')
    missing = [a for a, l in enumerate(grid_legs) if l is None]
    if len(missing) != 1:
        raise ValueError('can only derive one grid_leg')
    ax = missing[0]
    for a, l in enumerate(grid_legs):
        if l is not None and l.ind_len != shp[a]:
            raise ValueError('grid shape incompatible with grid_legs')
    chinfo = entries[0][1].chinfo
    qtotal = chinfo.make_valid(qtotal)
    qflat = [None] * shp[ax]
    for idx, e in entries:
        q = qtotal - e.qtotal
        for a, (i, l) in enumerate(zip(idx, grid_legs)):
            if a != ax:
                q = q - l.get_charge(l.get_qindex(i)[0]) * l.qconj
        q = chinfo.make_valid(q)
        i = idx[ax]
        if qflat[i] is None:
            qflat[i] = q
        elif np.any(qflat[i] != q):
            raise ValueError('different grid entries lead to different charges at index ' + str(i))
    if any(q is None for q in qflat):
        raise ValueError("can't derive flat charge for all indices:" + str(qflat))
    legs = list(grid_legs)
    legs[ax] = LegCharge.from_qflat(chinfo, chinfo.make_valid(qconj * np.array(qflat)), qconj)
    return legs


def grid_concat(grid, axes, copy=True):
    """block matrix of Arrays: concatenate the grid entries along `axes` (one per grid dimension; reference npc:3099).
    ``None`` entries are zero blocks."""
    npc = _npc()
    shp, entries = _grid_entries(grid)
    if len(shp) != len(axes):
        raise ValueError('need one axis per grid dimension')
    ref = entries[0][1]
    axes = ref.get_leg_indices(axes)
    lookup = dict(entries)
    # legs of the rows / columns of the grid
    grid_legs = []
    for gd, ax in enumerate(axes):
        legs_d = [None] * shp[gd]
        for idx, e in entries:
            if legs_d[idx[gd]] is None:
                legs_d[idx[gd]] = e.legs[ax]
        if any(l is None for l in legs_d):
            raise ValueError('a complete row/column of None entries in the grid')
        grid_legs.append(legs_d)

    def zero_entry(idx):
        legs = list(ref.legs)
        for gd, ax in enumerate(axes):
            legs[ax] = grid_legs[gd][idx[gd]]
        return npc.zeros(legs, ref.dtype, ref.qtotal, ref._labels)

    def build(prefix, gd):
        if gd == len(shp):
            return lookup.get(tuple(prefix)) or zero_entry(tuple(prefix))
        parts = [build(prefix + [i], gd + 1) for i in range(shp[gd])]
        return npc.concatenate(parts, axis=axes[gd], copy=copy)
    return build([], 0)


def detect_legcharge(flat_array, chargeinfo, legcharges, qtotal=None, qconj=+1, cutoff=None):
    """the one missing (``None``) LegCharge of a dense array from its non-zero entries (reference npc:3382)"""
    flat_array = np.asarray(flat_array)
    legs = list(legcharges)
    missing = [a for a, l in enumerate(legs) if l is None]
    if len(missing) != 1:
        raise ValueError('can only derive one leg')
    ax = missing[0]
    if cutoff is None:
        cutoff = QCUTOFF
    qtotal = chargeinfo.make_valid(qtotal)
    n = flat_array.shape[ax]
    moved = np.moveaxis(flat_array, ax, 0)
    qflat = np.zeros((n, chargeinfo.qnumber), dtype=QTYPE)
    other_legs = [l for a, l in enumerate(legs) if a != ax]
    for i in range(n):
        sub = moved[i]
        if sub.ndim == 0:
            q = qtotal.copy()
        else:
            pos = np.unravel_index(np.argmax(np.abs(sub)), sub.shape)
            if np.abs(sub[pos]) <= cutoff:
                q = np.zeros(chargeinfo.qnumber, QTYPE)
                qflat[i] = q
                continue
            q = qtotal.copy()
            for l, j in zip(other_legs, pos):
                q = q - l.get_charge(l.get_qindex(int(j))[0]) * l.qconj
        qflat[i] = chargeinfo.make_valid(q * qconj)
    legs[ax] = LegCharge.from_qflat(chargeinfo, qflat, qconj).bunch()[1]
    return legs


# ------------------------------------------------------------------------------------------------ small factorizations
def expm(a):
    """matrix exponential of a square (charge-blocked) matrix (reference npc:4288).  Real symmetric input (imaginary-time
    gates ``exp(-tau H_bond)``, tebd.py:446): ``V exp(w) V^T`` from the device `eigh`.  Other input: per block on the
    host with scipy (the gates are (d^2 x d^2) matrices built once per time step size)."""
    npc = _npc()
    if a.rank != 2:
        raise ValueError('expm needs a rank-2 Array')
    if a.dtype.kind != 'c':
        sym = npc.norm(a - a.conj().itranspose().iset_leg_labels(a._labels)) <= 1e-13 * max(npc.norm(a), 1e-300) \
            if a.legs[0].ind_len == a.legs[1].ind_len else False
        try:
            if sym:
                w, v = npc.eigh(a)
                res = npc.tensordot(v.scale_axis(np.exp(w), 1), v.conj(), axes=[1, 1])
                return res.iset_leg_labels(a._labels)
        except Exception:
            pass
    import scipy.linalg
    piped, b = a.as_completely_blocked()
    if isinstance(b, npc.ComplexArray):
        dense = scipy.linalg.expm(b.to_ndarray())
        res = npc.ComplexArray.from_ndarray(dense, b.legs, qtotal=b.qtotal, cutoff=0., labels=b._labels)
    else:
        if np.any(b.qtotal != 0):
            raise ValueError('expm of a matrix with non-zero total charge')
        blocks = [scipy.linalg.expm(blk) for blk in b.get_blocks_host()]
        qd = b._layout.qdata
        # blocks that are not stored are zero -> exp = identity on those sectors
        have = set(int(q) for q in qd[:, 0])
        extra_q, extra_b = [], []
        for qi, n in enumerate(b.legs[0].get_block_sizes()):
            if qi not in have:
                qj = b.legs[1].get_qindex_of_charges(b.legs[0].get_charge(qi) * b.legs[0].qconj * (-b.legs[1].qconj))
                extra_q.append([qi, int(qj)])
                extra_b.append(np.eye(int(n)))
        qd_all = np.concatenate([qd, np.array(extra_q, dtype=np.int64).reshape(-1, 2)]) if extra_q else qd
        res = npc.Array.from_blocks(b.legs, qd_all, blocks + extra_b, b.qtotal, b._labels)
    for ax in sorted(piped, reverse=True):
        res = res.split_legs(ax)
    return res.iset_leg_labels(a._labels)


def _not_on_device(name, ref):
    def f(*args, **kwargs):
        raise NotImplementedError('npc.{0} (reference {1}) is outside the two-site DMRG / TEBD path and is not provided by '
                                  'tenpy_b200'.format(name, ref))
    f.__name__ = name
    return f


eig = _not_on_device('eig', 'np_conserved.py:3959')
eigvals = _not_on_device('eigvals', 'np_conserved.py:4049')
speigs = _not_on_device('speigs', 'np_conserved.py:4078')
polar = _not_on_device('polar', 'np_conserved.py:4397')
orthogonal_columns = _not_on_device('orthogonal_columns', 'np_conserved.py:4330')


def lq(a, mode='reduced', inner_labels=[None, None], cutoff=None, pos_diag_L=False, qtotal_Q=None, inner_qconj=+1):
    """L-Q decomposition through :func:`qr` of the transpose (reference npc:4259)"""
    npc = _npc()
    label_L, label_Q = inner_labels
    Q, R = npc.qr(a.transpose(), mode=mode, inner_labels=[label_Q, label_L], cutoff=cutoff, pos_diag_R=pos_diag_L,
                  qtotal_Q=qtotal_Q, inner_qconj=-inner_qconj)
    return R.itranspose(), Q.itranspose()
