"""The remaining B1 surface of the DMRG/TEBD path (SURVEY.md section 8b): Array.take_slice / add_leg / extend,
npc.concatenate and small helpers, against golden vectors produced by the unmodified reference
(tests/golden/make_golden_b1.py).  Integer work (legs, block tables, qtotal) bit-exact, block data exact (pure copies)."""
import numpy as np
import pytest

import helpers as h


def _leg_from(g, prefix, chinfo):
    from tenpy_b200.linalg.charges import LegCharge
    return LegCharge.from_qind(chinfo, g[prefix + '_slices'], g[prefix + '_charges'], int(g[prefix + '_qconj']))


def _check_b1_ops():
    from tenpy_b200.linalg import np_conserved as npc
    g = h.load('b1_ops.npz')
    for case in range(int(g['n_cases'])):
        pre = 'c%d_' % case
        a = h.to_product(h.oarray_from(g, pre + 'a'))
        chinfo = a.chinfo
        # take_slice
        r = a.take_slice(int(g[pre + 'ts1_idx']), 'b')
        h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + 'ts1'), 0.)
        assert r.get_leg_labels() == ['a', 'c', 'd']
        r = a.take_slice([int(x) for x in g[pre + 'ts2_idx']], ['a', 'd'])
        h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + 'ts2'), 0.)
        # add_leg and its inverse
        new_leg = _leg_from(g, pre + 'al_leg', chinfo)
        j = int(g[pre + 'al_idx'])
        for axis, key in ((2, 'al2'), (0, 'al0')):
            r = a.add_leg(new_leg, j, axis=axis, label='n')
            h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + key), 0.)
            back = r.take_slice(j, 'n')
            h.assert_close(h.to_oracle(back), h.to_oracle(a), 0.)
        with pytest.raises(ValueError):
            a.add_leg(new_leg, j, axis=1, label='a')
        # extend
        r = a.extend('c', _leg_from(g, pre + 'ext_leg', chinfo))
        h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + 'ext'), 0.)
        r = a.extend('b', 2)
        h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + 'exti'), 0.)
        # concatenate
        b = h.to_product(h.oarray_from(g, pre + 'b'))
        c = h.to_product(h.oarray_from(g, pre + 'c'))
        r = npc.concatenate([a, b, c], axis='b')
        h.assert_close(h.to_oracle(r), h.oarray_from(g, pre + 'cat'), 0.)
        assert np.array_equal(r.to_ndarray(), np.concatenate([a.to_ndarray(), b.to_ndarray(), c.to_ndarray()], axis=1))
        with pytest.raises(ValueError):
            npc.concatenate([a, b.transpose(['b', 'a', 'c', 'd'])], axis='b')
        # small helpers
        assert a.is_completely_blocked() == all(l.is_blocked() for l in a.legs)
        sw = a.copy(deep=True).iswapaxes('a', 'c')
        assert np.array_equal(sw.to_ndarray(), np.swapaxes(a.to_ndarray(), 0, 2))
        o = npc.ones(a.legs, qtotal=a.qtotal)
        assert o._layout.same_blocks(a._layout) and np.all(np.concatenate(o.get_blocks_host(), axis=None) == 1.)
        assert np.array_equal(npc.detect_qtotal(a.to_ndarray(), a.legs), a.qtotal)


def _check_qr():
    """npc.qr per charge block against the reference's QR with pos_diag_R=True (unique for full-rank blocks): legs and
    block tables exact, entries to 1e-12; plus Q isometric, R upper triangular, Q R = A for ragged / deficient input"""
    from tenpy_b200.linalg import np_conserved as npc
    g = h.load('b1_ops.npz')
    for case in range(int(g['n_cases'])):
        pre = 'c%d_' % case
        for key, kw in (('', {}), ('q', None)):
            mat = h.to_product(h.oarray_from(g, pre + 'qr_m' + key))
            if kw is None:
                kw = dict(qtotal_Q=mat.qtotal, inner_qconj=-1)
            Q, R = npc.qr(mat, inner_labels=['q', 'r'], pos_diag_R=True, **kw)
            h.assert_close(h.to_oracle(Q), h.oarray_from(g, pre + 'qr_Q' + key), 1e-12)
            h.assert_close(h.to_oracle(R), h.oarray_from(g, pre + 'qr_R' + key), 1e-12)
            assert npc.norm(npc.tensordot(Q, R, axes=1) - mat) < 1e-13 * npc.norm(mat)
    rng = np.random.default_rng(7)
    for shape in [(7, 4), (4, 7), (1, 3), (3, 1), (33, 20)]:
        A = rng.standard_normal(shape)
        Q, R = npc.qr(npc.Array.from_ndarray_trivial(A))
        q, r = Q.to_ndarray(), R.to_ndarray()
        kk = min(shape)
        assert np.max(np.abs(q @ r - A)) < 1e-13 * np.abs(A).max() * max(shape)
        assert np.max(np.abs(q.T @ q - np.eye(kk))) < 1e-13
        assert np.all(np.tril(r, -1) == 0.) and np.all(np.diag(r) > 0.)
    A = rng.standard_normal((12, 3)) @ rng.standard_normal((3, 8))            # rank 3: dependent columns are replaced
    Q, R = npc.qr(npc.Array.from_ndarray_trivial(A))
    q, r = Q.to_ndarray(), R.to_ndarray()
    assert np.max(np.abs(q @ r - A)) < 1e-13 * np.abs(A).max() * 12 and np.max(np.abs(q.T @ q - np.eye(8))) < 1e-13
    with pytest.raises(NotImplementedError):
        npc.qr(npc.Array.from_ndarray_trivial(A), mode='complete')


def test_qr_host_logic(fake_device):
    _check_qr()


def test_qr_block_size_route_host_logic(fake_device):
    """npc.qr of an Array with one block of at most QR_HOUSEHOLDER_MAX rows and columns and one above: the small block goes
    through b200_block_qr_f64, the large one through Gram-Schmidt; both give numpy's factors (diagonal of R made
    non-negative) to the tolerances of _check_qr"""
    from tenpy_b200.linalg import np_conserved as npc
    ci = npc.ChargeInfo([1], ['N'])
    lL = npc.LegCharge.from_qind(ci, [0, 7, 407], [[0], [1]], +1)
    lR = npc.LegCharge.from_qind(ci, [0, 5, 8], [[0], [1]], -1)
    rng = np.random.default_rng(8)
    blocks = [rng.standard_normal((7, 5)), rng.standard_normal((400, 3))]
    assert max(blocks[0].shape) <= npc.QR_HOUSEHOLDER_MAX < max(blocks[1].shape)
    a = npc.Array.from_blocks([lL, lR], [[0, 0], [1, 1]], blocks, None, ['a', 'b'])
    n_qr, n_cols = fake_device.calls.get('block_qr', 0), npc.qr_stats['columns']
    Q, R = npc.qr(a, inner_labels=['q', 'r'])
    assert fake_device.calls.get('block_qr', 0) == n_qr + 1        # the small block: one Householder launch
    assert npc.qr_stats['columns'] == n_cols + 3                    # the large block: Gram-Schmidt, 3 columns
    q, r = Q.to_ndarray(), R.to_ndarray()
    rows, cols, segs = a.legs[0].slices, a.legs[1].slices, Q.legs[1].slices
    for i, A in enumerate(blocks):
        qb = q[rows[i]:rows[i + 1], segs[i]:segs[i + 1]]
        rb = r[segs[i]:segs[i + 1], cols[i]:cols[i + 1]]
        qq, rr = np.linalg.qr(A)
        sgn = np.where(np.diag(rr) < 0., -1., 1.)
        assert np.max(np.abs(qb - qq * sgn[None, :])) < 1e-12 and np.max(np.abs(rb - rr * sgn[:, None])) < 1e-12, i
        assert np.max(np.abs(qb @ rb - A)) < 1e-13 * np.abs(A).max() * max(A.shape), i
        assert np.max(np.abs(qb.T @ qb - np.eye(min(A.shape)))) < 1e-13, i
        assert np.all(np.tril(rb, -1) == 0.) and np.all(np.diag(rb) > 0.), i


@pytest.mark.gpu
def test_qr_gpu(gpu_lib):
    _check_qr()


def test_b1_ops_host_logic(fake_device):
    _check_b1_ops()


@pytest.mark.gpu
def test_b1_ops_gpu(gpu_lib):
    _check_b1_ops()
