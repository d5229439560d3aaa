"""Randomised differential test of the complex tensor layer (`ComplexArray`, tenpy_b200/linalg/_surface.py) against dense
complex128 NumPy, in the manner of tests/test_random_ops.py for the real Arrays: random charge rules (none, U(1),
U(1)xZ2, Z3), random legs (sorted or not, unbunched, ragged block sizes), random total charges incl. ones that allow no
block at all, and real and imaginary parts with different block tables.  Runs on the numpy test double with the complex
decompositions (tests/fake_device_complex.py) and, marked ``gpu``, on the CUDA kernels.

Reference rules:
* data movement, conjugation, sums and scaling by real factors or powers of two round once or not at all: they must
  match numpy exactly;
* products are compared with numpy in ``np.clongdouble``: ``|C - C_ref|_ij <= C_PROD k eps (|A||B|)_ij`` with k the
  number of summed terms (every complex product is a difference of two real FMA chains of k terms);
* decompositions use the bounds of tests/test_complex_decomp.py (p = max(m, n), k = min(m, n) of the dense matrix).

The module turns numpy's ComplexWarning into an error: a complex value cast silently to a real Array fails the test.
"""
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.filterwarnings('error::numpy.exceptions.ComplexWarning')

EPS = np.finfo(np.float64).eps
CLD = np.clongdouble
C_PROD = 4.
C_DEC = 32.
KINDS = ['both', 'im_subset', 'im_empty', 're_empty', 'im_zero', 're_zero']


@pytest.fixture
def fake_device_z():
    """the numpy test double of the device library with the complex decompositions (tests/fake_device_complex.py)"""
    import fake_device_complex
    lib, restore = fake_device_complex.install()
    yield lib
    restore()


# ---- random complex tensors ---------------------------------------------------------------------------------------------
def _rand_leg(rng, npc, chinfo, n, qconj):
    q = chinfo.make_valid(rng.integers(-2, 3, size=(n, chinfo.qnumber)))
    if chinfo.qnumber and rng.random() < 0.6:
        q = q[np.lexsort(q.T)]
    return npc.LegCharge.from_qflat(chinfo, q, qconj)


def _part(npc, full, keep):
    """the real Array `full` with only the blocks selected by `keep` (bool per stored block) stored"""
    qd = full._layout.qdata
    blocks = full.get_blocks_host()
    return npc.Array.from_blocks(full.legs, qd[keep], [b for b, k in zip(blocks, keep) if k], full.qtotal,
                                 full.get_leg_labels())


def _rand_complex(rng, npc, legs, qtotal, labels, kind):
    """ComplexArray on `legs`; `kind` picks the block tables of the parts:
    'both': re and im on every allowed block; 'im_subset': im on a random subset of the blocks of re; 'im_empty' / 're_empty':
    that part without blocks (purely real / purely imaginary); 'im_zero' / 're_zero': that part stores exactly zero blocks"""
    re = npc.Array.from_func(rng.standard_normal, legs, qtotal=qtotal, labels=labels)
    im = npc.Array.from_func(rng.standard_normal, legs, qtotal=qtotal, labels=labels)
    nb = re.stored_blocks
    if kind == 'im_subset':
        im = _part(npc, im, rng.random(nb) < 0.5)
    elif kind == 'im_empty':
        im = _part(npc, im, np.zeros(nb, bool))
    elif kind == 're_empty':
        re = _part(npc, re, np.zeros(nb, bool))
    elif kind == 'im_zero':
        im.iadd_prefactor_other(-1., im.copy())              # exactly zero blocks, still stored
    elif kind == 're_zero':
        re.iadd_prefactor_other(-1., re.copy())
    a = npc.ComplexArray(re, im)
    if kind in ('im_zero', 're_zero'):
        assert (a.im if kind == 'im_zero' else a.re).stored_blocks == nb
    return a


def _in_step(npc, x):
    """the wrapper and both parts agree on legs, labels, shape and total charge"""
    assert isinstance(x, npc.ComplexArray)
    x.test_sanity()
    for p in (x.re, x.im):
        assert type(p) is npc.Array
        assert p.get_leg_labels() == x.get_leg_labels()
        assert p.shape == x.shape and p.rank == x.rank
        assert np.array_equal(p.qtotal, x.qtotal)
        for lp, lx in zip(p.legs, x.legs):
            lp.test_equal(lx)
            assert lp.qconj == lx.qconj


def _exact(x, ref):
    got = x.to_ndarray()
    assert got.shape == ref.shape and np.array_equal(got, ref), np.max(np.abs(got - ref), initial=0.)


def _assert_product(got, ref, den, k, what=''):
    """componentwise product bound against the clongdouble reference"""
    err = np.abs(np.asarray(got) - ref)
    bound = C_PROD * max(k, 1) * EPS * den
    assert np.all(err <= bound), (what, float(np.max(err - bound)))


def _tdot_ref(A, B, axes):
    return (np.tensordot(A.astype(CLD), B.astype(CLD), axes=axes),
            np.tensordot(np.abs(A).astype(np.longdouble), np.abs(B).astype(np.longdouble), axes=axes))


# ---- the randomised check ------------------------------------------------------------------------------------------------
def _check_complex_ops(kind, n_cases=8):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(20261017 + KINDS.index(kind))
    chinfos = [npc.ChargeInfo(), npc.ChargeInfo([1], ['N']), npc.ChargeInfo([1, 2], ['N', 'P']), npc.ChargeInfo([3], ['Z3'])]
    labels = ['a', 'b', 'c', 'd']
    for case in range(n_cases):
        ci = chinfos[case % len(chinfos)]
        dims = [int(x) for x in rng.integers(1, 7, size=4)]
        legs = [_rand_leg(rng, npc, ci, d, int(rng.choice([-1, 1]))) for d in dims]
        qtot = ci.make_valid(rng.integers(-1, 2, size=ci.qnumber)) if rng.random() < 0.5 else None
        a = _rand_complex(rng, npc, legs, qtot, labels, kind)
        _in_step(npc, a)
        A = a.to_ndarray()
        assert A.dtype == np.complex128
        if kind in ('im_empty', 'im_zero'):
            assert not np.any(A.imag)
        if kind in ('re_empty', 're_zero'):
            assert not np.any(A.real)

        # --- data movement: exact
        perm = [int(x) for x in rng.permutation(4)]
        t = a.transpose(perm)
        _in_step(npc, t)
        _exact(t, A.transpose(perm))
        assert t.get_leg_labels() == [labels[p] for p in perm]
        t.itranspose(labels)
        _in_step(npc, t)
        _exact(t, A)
        i, j = (int(x) for x in rng.choice(4, size=2, replace=False))
        sw = a.copy()
        sw.iswapaxes(i, j)
        _in_step(npc, sw)
        _exact(sw, np.swapaxes(A, i, j))
        assert sw.isort_qdata() is sw
        _exact(sw, np.swapaxes(A, i, j))

        # --- combine / split, with and without a given pipe
        la_, lb_ = labels[i], labels[j]
        c = a.combine_legs([la_, lb_])
        _in_step(npc, c)
        pipe = c.get_leg('(%s.%s)' % (la_, lb_))
        rest = [x for x in range(4) if x not in (i, j)]
        dense_c = A.transpose([i, j] + rest).reshape((dims[i] * dims[j],) + tuple(dims[r] for r in rest))
        flat = np.array([pipe.map_incoming_flat([x, y]) for x in range(dims[i]) for y in range(dims[j])])
        pos = c.get_leg_index('(%s.%s)' % (la_, lb_))
        assert np.array_equal(np.moveaxis(c.to_ndarray(), pos, 0)[flat], dense_c)
        back = c.split_legs()
        _in_step(npc, back)
        _exact(back.itranspose(labels), A)
        given = a.make_pipe([la_, lb_])
        c2 = a.combine_legs([la_, lb_], pipes=given)
        _in_step(npc, c2)
        assert c2.legs[c2.get_leg_index('(%s.%s)' % (la_, lb_))] is given
        _exact(c2, c.to_ndarray())
        _exact(c2.split_legs(pos).itranspose(labels), A)

        # --- slices, projections, new legs
        ax = int(rng.integers(0, 4))
        idx = int(rng.integers(0, dims[ax]))
        ts = a.take_slice(idx, ax)
        _in_step(npc, ts)
        _exact(ts, np.take(A, idx, axis=ax))
        if ax != 3:
            idx2 = int(rng.integers(0, dims[3]))
            ts2 = a.take_slice([idx, idx2], [labels[ax], 'd'])
            _in_step(npc, ts2)
            _exact(ts2, np.take(np.take(A, idx2, axis=3), idx, axis=ax))
        mask = rng.random(dims[ax]) < 0.6
        mask[int(rng.integers(0, dims[ax]))] = True
        pr = a.copy()
        ret = pr.iproject(mask, ax)
        _in_step(npc, pr)
        _exact(pr, np.compress(mask, A, axis=ax))
        ref_ret = a.re.copy().iproject(mask, ax)
        assert np.array_equal(ret[0], ref_ret[0]) and all(np.array_equal(x, y) for x, y in zip(ret[1], ref_ret[1]))
        new_leg = _rand_leg(rng, npc, ci, 3, int(rng.choice([-1, 1])))
        jn = int(rng.integers(0, 3))
        al = a.add_leg(new_leg, jn, axis=ax, label='n')
        _in_step(npc, al)
        assert al.get_leg_labels()[ax] == 'n'
        _exact(al, np.expand_dims(A, ax) * (np.arange(3) == jn).reshape([3 if x == ax else 1 for x in range(5)]))
        tl = a.add_trivial_leg(axis=ax, label='t', qconj=int(rng.choice([-1, 1])))
        _in_step(npc, tl)
        _exact(tl, np.expand_dims(A, ax))
        sq = tl.squeeze('t')
        _in_step(npc, sq)
        _exact(sq, A)
        assert sq.get_leg_labels() == labels
        unit = _rand_leg(rng, npc, ci, 1, +1)
        sq2 = a.add_leg(unit, 0, axis=0, label='u').squeeze('u')
        _in_step(npc, sq2)
        _exact(sq2, A)
        assert np.array_equal(sq2.qtotal, a.qtotal)
        ext = a.extend(ax, int(rng.integers(1, 4)))
        _in_step(npc, ext)
        dense_ext = np.zeros(ext.shape, complex)
        dense_ext[tuple(slice(0, d) for d in dims)] = A
        _exact(ext, dense_ext)
        newq = ci.make_valid(rng.integers(-2, 3, size=ci.qnumber))
        g = a.gauge_total_charge(ax, newq)
        _in_step(npc, g)
        assert np.array_equal(g.qtotal, ci.make_valid(newq))
        _exact(g, A)

        # --- labels stay in step between the wrapper and both parts
        lab = a.copy()
        lab.ireplace_label('a', 'x')
        _in_step(npc, lab)
        lab.ireplace_labels(['b', 'c'], ['y', 'z'])
        _in_step(npc, lab)
        assert lab.get_leg_labels() == ['x', 'y', 'z', 'd']
        lab.idrop_labels(['y'])
        _in_step(npc, lab)
        assert lab.get_leg_labels() == ['x', None, 'z', 'd']
        lab.iset_leg_labels(['p', 'q', 'r', 's'])
        _in_step(npc, lab)
        rl = lab.replace_label('p', 'P').replace_labels(['q', 'r'], ['Q', 'R'])
        _in_step(npc, rl)
        assert rl.get_leg_labels() == ['P', 'Q', 'R', 's'] and lab.get_leg_labels() == ['p', 'q', 'r', 's']
        _exact(rl, A)

        # --- conjugation: exact values, flipped legs
        for cj in (a.conj(), a.copy().iconj()):
            _in_step(npc, cj)
            _exact(cj, A.conj())
            assert [l.qconj for l in cj.legs] == [-l.qconj for l in a.legs]
            assert cj.get_leg_labels() == ['a*', 'b*', 'c*', 'd*']
            assert np.array_equal(cj.qtotal, ci.make_valid(-a.qtotal))
        cc = a.complex_conj()
        _in_step(npc, cc)
        _exact(cc, A.conj())
        assert [l.qconj for l in cc.legs] == [l.qconj for l in a.legs] and cc.get_leg_labels() == labels
        nc = a.conj(complex_conj=False)
        _in_step(npc, nc)
        _exact(nc, A)
        assert [l.qconj for l in nc.legs] == [-l.qconj for l in a.legs]

        # --- scaling
        shp = [1] * 4
        shp[ax] = dims[ax]
        s_real = rng.standard_normal(dims[ax])
        s_cplx = rng.standard_normal(dims[ax]) + 1.j * rng.standard_normal(dims[ax])
        sc = a.scale_axis(s_real, ax)
        _in_step(npc, sc)
        _exact(sc, A * s_real.reshape(shp))
        for x in (a.scale_axis(s_cplx, ax), a.copy().iscale_axis(s_cplx, labels[ax])):
            _in_step(npc, x)
            _assert_product(x.to_ndarray(), A.astype(CLD) * s_cplx.astype(CLD).reshape(shp),
                            np.abs(A) * np.abs(s_cplx).reshape(shp), 1, 'scale_axis complex')
        _exact(a.copy().iscale_axis(s_real + 0.j, ax), A * s_real.reshape(shp))     # complex dtype, zero imaginary part
        for z in (2., -0.5, 2.j, -0.25j):
            x = a.copy()
            x.iscale_prefactor(z)
            _in_step(npc, x)
            _exact(x, A * z)
        for z in (0.3, 0.3 - 1.2j):
            x = a.copy().iscale_prefactor(z)
            _in_step(npc, x)
            _assert_product(x.to_ndarray(), A.astype(CLD) * CLD(z), np.abs(A) * abs(z), 1, 'iscale_prefactor')
        zero = a.copy().iscale_prefactor(0.)
        _exact(zero, np.zeros_like(A))

        # --- linear combinations with a complex / real partner on the same legs (own block tables)
        kind_b = KINDS[int(rng.integers(0, len(KINDS)))]
        b = _rand_complex(rng, npc, legs, a.qtotal, labels, kind_b)
        B = b.to_ndarray()
        for z in (1.5, 0.7 + 0.2j, -1.j):
            for other, O in ((b, B), (b.re, B.real)):
                x = a.copy().iadd_prefactor_other(z, other)
                _in_step(npc, x)
                _assert_product(x.to_ndarray(), A.astype(CLD) + CLD(z) * O.astype(CLD), np.abs(A) + abs(z) * np.abs(O), 2,
                                'iadd_prefactor_other')
        for x, ref in ((a + b, A + B), (a - b, A - B), (a + b.re, A + B.real), (b.re + a, B.real + A),
                       (a - b.re, A - B.real), (b.re - a, B.real - A), (-a, -A), (a / 2., A / 2.), (a / -0.25j, A / -0.25j)):
            _in_step(npc, x)
            _exact(x, ref)
        for x, ref in ((a / (1.5 - 0.5j), A / (1.5 - 0.5j)), (b.re / (0.5 + 2.j), B.real / (0.5 + 2.j))):
            _in_step(npc, x)
            _assert_product(x.to_ndarray(), ref.astype(CLD), 2. * np.abs(ref), 1, '/')
        x = a.copy()
        x += b
        x -= b.re
        _in_step(npc, x)
        _exact(x, (A + B) - B.real)

        # --- norm / inner
        assert abs(npc.norm(a) - np.linalg.norm(A)) <= C_PROD * A.size * EPS * np.linalg.norm(A)
        assert a.norm() == npc.norm(a)
        AL, BL = A.astype(CLD), B.astype(CLD)
        den = np.sum(np.abs(A) * np.abs(B))
        for do_conj in (True, False):
            for x, y, X, Y in ((a, b, AL, BL), (a.re, b, AL.real, BL), (a, b.re, AL, BL.real)):
                yy = y if do_conj else y.conj()
                val = npc.inner(x, yy, axes='range', do_conj=do_conj)
                ref = np.sum(X.conj() * Y) if do_conj else np.sum(X * Y.conj())
                assert isinstance(val, complex)
                _assert_product(val, ref, den, A.size, 'inner')
        assert isinstance(npc.inner(a, b, axes='labels', do_conj=True), complex)
        _assert_product(npc.inner(a, b, axes='labels', do_conj=True), np.sum(AL.conj() * BL), den, A.size, 'inner labels')

        # --- tensordot: all four real/complex operand pairs, and a full contraction to a complex scalar
        k1, k2 = (int(x) for x in rng.choice(4, size=2, replace=False))
        extra = [_rand_leg(rng, npc, ci, int(rng.integers(1, 5)), int(rng.choice([-1, 1]))) for _ in range(2)]
        d_legs = [extra[0], legs[k1].conj(), extra[1], legs[k2].conj()]
        d = _rand_complex(rng, npc, d_legs, ci.make_valid(rng.integers(-1, 2, size=ci.qnumber)), ['e', 'k1', 'f', 'k2'],
                          KINDS[int(rng.integers(0, len(KINDS)))])
        D = d.to_ndarray()
        kk = dims[k1] * dims[k2]
        for x, y, X, Y in ((a, d, A, D), (a.re, d, A.real, D), (a, d.re, A, D.real), (a.re, d.re, A.real, D.real)):
            r = npc.tensordot(x, y, axes=[[labels[k1], labels[k2]], ['k1', 'k2']])
            ref_t, den_t = _tdot_ref(X, Y, [[k1, k2], [1, 3]])
            if isinstance(x, npc.ComplexArray) or isinstance(y, npc.ComplexArray):
                _in_step(npc, r)
            else:
                assert type(r) is npc.Array
            _assert_product(r.to_ndarray(), ref_t, den_t, kk, 'tensordot')
        full = npc.tensordot(a, b.conj(), axes=[labels, [l + '*' for l in labels]])
        assert isinstance(full, complex)
        _assert_product(full, np.sum(AL * BL.conj()), den, A.size, 'full tensordot')
        full_r = npc.tensordot(b.conj(), a.re, axes=[[l + '*' for l in labels], labels])
        assert isinstance(full_r, complex)
        _assert_product(full_r, np.sum(BL.conj() * AL.real), den, A.size, 'full tensordot, real operand')

        # --- outer products and concatenation
        o = npc.outer(a.take_slice([0, 0], ['c', 'd']), d.re.take_slice([0, 0], ['e', 'f']))
        _in_step(npc, o)
        _exact(o, np.multiply.outer(A[:, :, 0, 0], D.real[0, :, 0, :]))
        legs2 = list(legs)
        legs2[ax] = _rand_leg(rng, npc, ci, int(rng.integers(1, 5)), legs[ax].qconj)
        e = _rand_complex(rng, npc, legs2, a.qtotal, labels, KINDS[int(rng.integers(0, len(KINDS)))])
        for parts, dense in (([a, e], [A, e.to_ndarray()]), ([a.re, e, a], [A.real, e.to_ndarray(), A])):
            cat = npc.concatenate(parts, axis=ax)
            _in_step(npc, cat)
            _exact(cat, np.concatenate(dense, axis=ax))

        # --- element access, comparison, types, pickling
        qd = np.unique(np.concatenate([a.re._layout.qdata, a.im._layout.qdata]), axis=0)
        for q in qd:
            blk = a.get_block(q)
            sl = tuple(l.get_slice(qi) for l, qi in zip(a.legs, q))
            assert np.array_equal(blk, A[sl])
        ix = tuple(int(rng.integers(0, n)) for n in dims)
        assert a[ix] == A[ix] and isinstance(a[ix], np.complex128)
        _exact(a[ix[0], :, ix[2]], A[ix[0], :, ix[2]])
        order = rng.permutation(dims[1])
        _exact(a[:, order], A[:, order])
        mask_d = rng.random(dims[3]) < 0.5
        mask_d[0] = True
        _exact(a[..., mask_d], A[..., mask_d])
        assert a == a.copy() and b.re.astype(np.complex128) == b.re
        if np.any(A.imag):
            assert not a == a.complex_conj()
        if np.any(A):
            assert not a == a * (1. + 1e-3j)
        ac = a.re.astype(np.complex128)
        _in_step(npc, ac)
        assert ac.im.stored_blocks == 0
        _exact(ac, A.real + 0.j)
        if np.any(A.imag):
            with pytest.warns(UserWarning, match='imaginary'):
                ar = a.astype(np.float64)
        else:
            ar = a.astype(np.float64)
        assert type(ar) is npc.Array and np.array_equal(ar.to_ndarray(), A.real)
        assert a.astype(np.complex128) is not a and a.astype(np.complex128, copy=False) is a
        pk = pickle.loads(pickle.dumps(a))
        _in_step(npc, pk)
        _exact(pk, A)

        # --- trace of a square matrix
        m = npc.ComplexArray(*(npc.Array.from_func(rng.standard_normal, [legs[0], legs[0].conj()], labels=['p', 'p*'])
                               for _ in range(2)))
        M = m.to_ndarray()
        tr = npc.trace(m)
        assert isinstance(tr, complex)
        _assert_product(tr, np.trace(M.astype(CLD)), np.sum(np.abs(np.diag(M))), dims[0], 'trace')

        # --- decompositions of the matrix (a b) x (c d)
        mat = a.combine_legs([['a', 'b'], ['c', 'd']], qconj=[+1, -1])
        if mat.stored_blocks:
            _check_decompositions(npc, mat)


def _check_decompositions(npc, mat):
    Md = mat.to_ndarray()
    mm, nn = Md.shape
    p, kmin = max(mm, nn), min(mm, nn)
    fro, n2 = np.linalg.norm(Md), np.linalg.norm(Md, 2)
    U, S, VH = npc.svd(mat, inner_labels=['x', 'x*'])
    assert isinstance(U, npc.ComplexArray) and isinstance(VH, npc.ComplexArray) and S.dtype == np.float64
    _in_step(npc, U)
    _in_step(npc, VH)
    u, vh = U.to_ndarray(), VH.to_ndarray()
    k = len(S)
    assert k <= kmin and np.all(S >= 0.)
    assert np.max(np.abs(u.conj().T @ u - np.eye(k))) <= C_DEC * max(k, 16) * EPS
    assert np.max(np.abs(vh @ vh.conj().T - np.eye(k))) <= C_DEC * max(k, 16) * EPS
    rec = npc.tensordot(U.scale_axis(S, 1), VH, axes=1)
    assert np.linalg.norm(rec.to_ndarray() - Md) <= C_DEC * p * EPS * fro
    s_ref = np.linalg.svd(Md, compute_uv=False)
    s_got = np.sort(S)[::-1]
    assert np.max(np.abs(s_got - s_ref[:k])) <= C_DEC * p * EPS * n2
    assert np.all(s_ref[k:] <= C_DEC * p * EPS * n2)
    Q, R = npc.qr(mat, inner_labels=['q', 'q*'])
    assert isinstance(Q, npc.ComplexArray) and isinstance(R, npc.ComplexArray)
    _in_step(npc, Q)
    _in_step(npc, R)
    q, r = Q.to_ndarray(), R.to_ndarray()
    assert np.max(np.abs(q.conj().T @ q - np.eye(q.shape[1]))) <= C_DEC * max(q.shape[1], 16) * EPS
    assert np.linalg.norm(q @ r - Md) <= C_DEC * p * EPS * fro
    for qi in np.unique(np.concatenate([R.re._layout.qdata, R.im._layout.qdata]), axis=0):
        d = np.diag(R.get_block(qi))
        assert np.all(d.imag == 0.) and np.all(d.real >= 0.), d


# ---- complex factors and values reaching real Arrays: a complex result or a TypeError, never a silent real part --------
def _legs_u1(npc):
    ci = npc.ChargeInfo([1], ['N'])
    return (npc.LegCharge.from_qflat(ci, [[0], [1], [0], [1], [2]], +1),
            npc.LegCharge.from_qflat(ci, [[1], [0], [1], [2]], -1))


def _check_complex_factors():
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(7)
    la, lb = _legs_u1(npc)
    r = npc.Array.from_func(rng.standard_normal, [la, lb], labels=['a', 'b'])
    R = r.to_ndarray()
    s = rng.standard_normal(4) + 1.j * rng.standard_normal(4)
    # scale_axis of a real Array: complex factors give a ComplexArray (re Re(s), re Im(s)), exactly
    x = r.scale_axis(s, 'b')
    _in_step(npc, x)
    _exact(x, R.real * s.real[None, :] + 1.j * (R.real * s.imag[None, :]))
    with pytest.raises(TypeError, match='scale_axis'):
        r.copy().iscale_axis(s, 'b')
    _exact(r.copy().iscale_axis(s.real + 0.j, 'b').astype(np.complex128), R * s.real[None, :])
    # ComplexArray.scale_axis / iscale_axis: (re + i im)(sr + i si)
    c = npc.ComplexArray(r, npc.Array.from_func(rng.standard_normal, [la, lb], labels=['a', 'b']))
    C = c.to_ndarray()
    for y in (c.scale_axis(s, 1), c.copy().iscale_axis(s, 'b')):
        _in_step(npc, y)
        _assert_product(y.to_ndarray(), C.astype(CLD) * s.astype(CLD)[None, :], np.abs(C) * np.abs(s)[None, :], 1)
    # diag
    d = rng.standard_normal(5) + 1.j * rng.standard_normal(5)
    for dd in (d, 1.5 - 2.j):
        x = npc.diag(dd, la, labels=['p', 'p*'])
        _in_step(npc, x)
        _exact(x, np.diag(d) if np.ndim(dd) else dd * np.eye(5))
    assert type(npc.diag(d.real, la)) is npc.Array
    # from_func with complex blocks dispatches like from_blocks
    x = npc.Array.from_func(lambda shape: rng.standard_normal(shape) + 1.j * rng.standard_normal(shape), [la, lb])
    _in_step(npc, x)
    assert np.any(x.to_ndarray().imag) and np.any(x.to_ndarray().real)
    assert type(npc.Array.from_func(np.ones, [la, lb])) is npc.Array
    # astype
    x = r.astype(np.complex128)
    _in_step(npc, x)
    assert x.im.stored_blocks == 0
    _exact(x, R + 0.j)
    with pytest.raises(NotImplementedError):
        r.astype(np.float32)
    # in-place updates of a real Array can not take complex data
    with pytest.raises(TypeError, match='self \\+ prefactor \\* other'):
        r.copy().iadd_prefactor_other(1.j, r)
    with pytest.raises(TypeError, match='self \\+ prefactor \\* other'):
        r.copy().iadd_prefactor_other(1., c)
    _exact(r + 1.j * r, R * (1. + 1.j))
    blk = r.copy().get_block([0, 0])
    with pytest.raises(TypeError):
        blk[0, 0] = 1. + 2.j
    i, j = (int(v) for v in np.argwhere(R != 0.)[0])                # an entry of an allowed block
    y = r.copy()
    with pytest.raises(TypeError):
        y[i, j] = 1. + 2.j
    y = c.copy()
    y[i, j] = 1. + 2.j
    C2 = C.copy()
    C2[i, j] = 1. + 2.j
    _exact(y, C2)
    # indexing with an unsorted index array (real and complex)
    for idx in ([2, 0, 1], [3, 1, 0, 2], [1, 0]):
        assert np.array_equal(r[:, idx].to_ndarray(), R[:, idx])
        _exact(c[:, idx], C[:, idx])


def _check_expm():
    import scipy.linalg
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(8)
    ci = npc.ChargeInfo([1], ['N'])
    leg = npc.LegCharge.from_qflat(ci, [[0], [1], [0], [2], [1], [1], [0]], +1)
    n = leg.ind_len
    q = leg.to_qflat()[:, 0]
    mask = np.equal.outer(q, q)
    h = (rng.standard_normal((n, n)) + 1.j * rng.standard_normal((n, n))) * mask
    herm = 0.5 * (h + h.conj().T)
    sym = 0.5 * (h.real + h.real.T)

    def check(x, ref, gen):
        bound = C_DEC * n * EPS * np.linalg.norm(ref, 2) * max(1., np.linalg.norm(gen, 2))
        assert np.max(np.abs(x.to_ndarray() - ref)) <= bound
    for gen in (0.7 * h, -0.1j * herm):                              # a complex gate; exp(-i dt H) with a Hermitian H
        g = npc.Array.from_ndarray(gen, [leg, leg.conj()], labels=['p', 'p*'])
        assert isinstance(g, npc.ComplexArray)
        u = npc.expm(g)
        _in_step(npc, u)
        assert u.get_leg_labels() == ['p', 'p*']
        check(u, scipy.linalg.expm(gen), gen)
    ud = npc.expm(npc.Array.from_ndarray(-0.1j * herm, [leg, leg.conj()])).to_ndarray()
    assert np.max(np.abs(ud @ ud.conj().T - np.eye(n))) <= C_DEC * n * EPS
    for gen in (sym, h.real):                                        # real symmetric (device eigh), real non-symmetric
        g = npc.Array.from_ndarray(gen, [leg, leg.conj()], labels=['p', 'p*'])
        u = npc.expm(g)
        assert type(u) is npc.Array and u.get_leg_labels() == ['p', 'p*']
        check(u, scipy.linalg.expm(gen), gen)


def test_complex_factors_fake(fake_device_z):
    _check_complex_factors()


def test_expm_fake(fake_device_z):
    calls = fake_device_z.calls.get('block_eigh', 0)
    _check_expm()
    assert fake_device_z.calls.get('block_eigh', 0) > calls        # the real symmetric generator took the eigh route


@pytest.mark.gpu
def test_complex_factors_gpu(gpu_lib):
    _check_complex_factors()


@pytest.mark.gpu
def test_expm_gpu(gpu_lib):
    _check_expm()


# ---- the kernel paths of the four real products of a complex contraction (GPU) --------------------------------------------
# A[L, K*] . B[K, R*], block diagonal in a U(1) charge c; per charge (m, [k of the K blocks of that charge], n).  The grouped
# GEMM picks per output block: 64x64 tiles by default, 32x32 tiles when they waste less than 70 % of the 64x64 area,
# thin_n for n <= 8 with m >= 4 n and k-sum <= 64, thin_m for m <= 8 with n >= 4 m and k-sum <= 64; the VEC variants of
# the tile kernels run when every n and k of the launch is even, the scalar variants otherwise.  K is unbunched and
# unsorted: two K blocks of one charge feed one output block through two block pairs.
TDOT_PATHS = {
    # all extents even: every launch on the VEC tile kernels
    'even': [(128, [64, 64], 128),     # 64x64 tiles, two block pairs
             (96, [40], 96),           # 32x32 tiles
             (300, [40], 8),           # thin_n
             (6, [2, 10], 256),        # thin_m, two block pairs
             (2, [2], 2)],             # 32x32, one partial tile
    # odd extents: every launch on the scalar tile kernels
    'odd': [(129, [63, 1], 127),       # 64x64 tiles with ragged edges, two block pairs (one of k = 1)
            (95, [33], 17),            # 32x32 tiles
            (257, [1, 3], 7),          # thin_n, two block pairs
            (5, [61], 300),            # thin_m
            (1, [1], 1)],              # 32x32, a 1x1 block
}


def _check_tdot_paths(case):
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(len(case))
    spec = TDOT_PATHS[case]
    ci = npc.ChargeInfo([1], ['N'])

    def leg(sizes, charges):
        return npc.LegCharge.from_qind(ci, np.concatenate(([0], np.cumsum(sizes))), np.array(charges).reshape(-1, 1), +1)
    L = leg([m for m, _, _ in spec], range(len(spec)))
    R = leg([n for _, _, n in spec], range(len(spec)))
    kb = [(k, c) for c, (_, ks, _) in enumerate(spec) for k in ks]
    kb = [kb[i] for i in rng.permutation(len(kb))]
    K = leg([k for k, _ in kb], [c for _, c in kb])
    a = _rand_complex(rng, npc, [L, K.conj()], None, ['l', 'k*'], 'im_subset')
    b = _rand_complex(rng, npc, [K, R.conj()], None, ['k', 'r*'], 'both')
    A, B = a.to_ndarray(), b.to_ndarray()
    qL, qK, qR = (x.to_qflat()[:, 0] for x in (L, K, R))
    for x, y, X, Y in ((a, b, A, B), (a.re, b, A.real, B), (a, b.re, A, B.real)):
        got = npc.tensordot(x, y, axes=['k*', 'k'])
        _in_step(npc, got)
        got = got.to_ndarray()
        ref = np.zeros(got.shape, CLD)
        bound = np.zeros(got.shape)
        for c, (_, ks, _) in enumerate(spec):
            ri, ki, cj = np.nonzero(qL == c)[0], np.nonzero(qK == c)[0], np.nonzero(qR == c)[0]
            xb, yb = X[np.ix_(ri, ki)], Y[np.ix_(ki, cj)]
            ref[np.ix_(ri, cj)] = xb.astype(CLD) @ yb.astype(CLD)
            bound[np.ix_(ri, cj)] = C_PROD * sum(ks) * EPS * (np.abs(xb) @ np.abs(yb))
        assert np.all(np.abs(got - ref) <= bound), (case, float(np.max(np.abs(got - ref) - bound)))


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(TDOT_PATHS))
def test_complex_tensordot_paths_gpu(gpu_lib, case):
    _check_tdot_paths(case)


@pytest.mark.parametrize('kind', KINDS)
def test_complex_ops_fake(fake_device_z, kind):
    _check_complex_ops(kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_complex_ops_gpu(gpu_lib, kind):
    _check_complex_ops(kind)
