"""npc.svd, npc.qr and npc.eigh of charge-conserving Arrays whose blocks lie far apart in scale (1e-200, 1e-120, 1,
1e+200), checked block by block against dense numpy.  Every bound is relative to the block it concerns: a result that is
only right relative to the norm of the whole Array is wrong for its small blocks.

The same cases run on the numpy test double (``fake_device``: the host logic, including the completion of deflated
directions and the Gram-Schmidt QR of blocks above 384) and on the GPU."""
import numpy as np
import pytest

from fake_device import fro_norm

EPS = np.finfo(np.float64).eps


def _legs(npc, big):
    """two legs with five sectors; sector 4 is 400 long when `big` (a block above QR_HOUSEHOLDER_MAX), else 3"""
    ci = npc.ChargeInfo([1], ['N'])
    last = 400 if big else 3
    lL = npc.LegCharge.from_qind(ci, np.cumsum([0, 6, 8, 8, 8, last]), [[0], [1], [2], [3], [4]], +1)
    lR = npc.LegCharge.from_qind(ci, np.cumsum([0, 5, 9, 6, 7, last]), [[0], [1], [2], [3], [4]], -1)
    return lL, lR


def _low_rank(rng, m, n, r):
    return rng.standard_normal((m, r)) @ rng.standard_normal((r, n))


def _scaled_blocks(rng, lL, lR, big):
    """diagonal blocks: 6x5 at 1e-200, 8x9 at 1, 8x6 at 1e+200, a rank-2 8x7 block at 1e-120, the last at 1e-200"""
    shapes = list(zip(lL.get_block_sizes(), lR.get_block_sizes()))
    blocks = [1e-200 * rng.standard_normal(shapes[0]), rng.standard_normal(shapes[1]),
              1e+200 * rng.standard_normal(shapes[2]), 1e-120 * _low_rank(rng, *shapes[3], 2),
              1e-200 * rng.standard_normal(shapes[4])]
    return [[i, i] for i in range(5)], blocks


def _array(npc, rng, big=False):
    lL, lR = _legs(npc, big)
    qd, blocks = _scaled_blocks(rng, lL, lR, big)
    return npc.Array.from_blocks([lL, lR], qd, blocks, None, ['a', 'b']), blocks


def _svd_case():
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(5)
    a, blocks = _array(npc, rng)
    U, S, VH = npc.svd(a, inner_labels=['i', 'i*'])
    u, vh = U.to_ndarray(), VH.to_ndarray()
    kk = len(S)
    assert kk == sum(min(b.shape) for b in blocks)
    assert np.max(np.abs(u.T @ u - np.eye(kk))) <= 32 * EPS * kk      # isometries: |U^T U - 1| <= 32 eps k
    assert np.max(np.abs(vh @ vh.T - np.eye(kk))) <= 32 * EPS * kk
    rows, cols, segs = a.legs[0].slices, a.legs[1].slices, VH.legs[0].slices
    for i, blk in enumerate(blocks):
        m, n = blk.shape
        s = S[segs[i]:segs[i + 1]]
        ub = u[rows[i]:rows[i + 1], segs[i]:segs[i + 1]]
        vb = vh[segs[i]:segs[i + 1], cols[i]:cols[i + 1]]
        fro = fro_norm(blk)
        s_ref = np.linalg.svd(blk, compute_uv=False)
        rank = int(np.sum(s_ref > 16 * EPS * max(m, n) * fro))
        # per block: S to 8 max(m, n) eps |A_i|_F of LAPACK, reconstruction to 8 max(m, n) eps |A_i|_F
        assert np.max(np.abs(np.sort(s)[::-1][:rank] - s_ref[:rank])) <= 8 * max(m, n) * EPS * fro, (i, s, s_ref)
        assert np.max(np.abs((ub * s) @ vb - blk)) <= 8 * max(m, n) * EPS * fro, i
        genuine = s[:rank]
        completed = s[rank:]
        # completed directions of a rank-deficient block: positive, and never above the block's genuine singular values,
        # so that a truncation keeps the genuine ones first at any scale
        assert np.all(completed > 0.) and np.all(completed <= genuine.min()), (i, genuine, completed)


def _qr_case():
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(6)
    a, blocks = _array(npc, rng, big=True)
    Q, R = npc.qr(a, inner_labels=['q', 'q*'])
    q, r = Q.to_ndarray(), R.to_ndarray()
    k = q.shape[1]
    assert np.max(np.abs(q.T @ q - np.eye(k))) <= 8 * EPS * 400      # |Q^T Q - 1| <= 8 eps max(m)
    rows, cols, segs = a.legs[0].slices, a.legs[1].slices, Q.legs[1].slices
    for i, blk in enumerate(blocks):
        m, n = blk.shape
        qb = q[rows[i]:rows[i + 1], segs[i]:segs[i + 1]]
        rb = r[segs[i]:segs[i + 1], cols[i]:cols[i + 1]]
        fro = fro_norm(blk)
        # per block: |Q_i R_i - A_i| <= 8 max(m, n) eps |A_i|_F, R_i upper triangular with a non-negative diagonal
        assert np.max(np.abs(qb @ rb - blk)) <= 8 * max(m, n) * EPS * fro, i
        assert np.all(np.tril(rb, -1) == 0.) and np.all(np.diag(rb) >= 0.), i


def _eigh_case():
    from tenpy_b200.linalg import np_conserved as npc
    rng = np.random.default_rng(7)
    lL, _ = _legs(npc, False)
    sizes = lL.get_block_sizes()
    blocks = []
    for sz, sc in zip(sizes, [1e-200, 1., 1e+200, 1e-120, 1e-200]):
        x = rng.standard_normal((sz, sz))
        blocks.append(sc * (x + x.T))
    a = npc.Array.from_blocks([lL, lL.conj()], [[i, i] for i in range(5)], blocks, None, ['p', 'p*'])
    W, V = npc.eigh(a)
    v = V.to_ndarray()
    assert np.max(np.abs(v.T @ v - np.eye(len(W)))) <= 16 * EPS * 16      # |V^T V - 1| <= 16 eps max(n, 16)
    sl = lL.slices
    for i, blk in enumerate(blocks):
        n = blk.shape[0]
        p = max(n, 16)
        fro = fro_norm(blk)
        w, vb = W[sl[i]:sl[i + 1]], v[sl[i]:sl[i + 1], sl[i]:sl[i + 1]]
        # per block (test_gpu_kernel_edges._check_eigh): eigenvalues and residual to 2 p eps |A_i|_F, p = max(n, 16)
        assert np.max(np.abs(w - np.linalg.eigvalsh(blk))) <= 2 * p * EPS * fro, (i, w)
        assert np.max(np.abs(blk @ vb - vb * w)) <= 2 * p * EPS * fro, i


def test_npc_svd_scale_range_fake(fake_device):
    _svd_case()


def test_npc_qr_scale_range_fake(fake_device):
    _qr_case()


def test_npc_eigh_scale_range_fake(fake_device):
    _eigh_case()


@pytest.mark.gpu
def test_npc_svd_scale_range_gpu(gpu_lib):
    _svd_case()


@pytest.mark.gpu
def test_npc_qr_scale_range_gpu(gpu_lib):
    _qr_case()


@pytest.mark.gpu
def test_npc_eigh_scale_range_gpu(gpu_lib):
    _eigh_case()
