"""npc.qr on rank-deficient, nearly dependent, ill-conditioned, zero and badly scaled blocks, on each of its routes.

npc.qr picks the route from the block alone: real blocks of up to QR_HOUSEHOLDER_MAX = 384 rows and columns go to the
Householder kernel b200_block_qr_f64, larger real blocks to the Gram-Schmidt composition _block_qr_cgs2, complex blocks of
every size to b200_block_qr_z.  Every input is one charged Array whose diagonal blocks have the shapes of SHAPES, on both
sides of the cut-off, so that one npc.qr call runs both real routes.  The same inputs made complex, (1 + 2i) A + i A' with A'
an independent draw of the same structure (the same dependencies, zero columns and scales), run through the complex kernel.

Input classes (seeded):
* exact_rank: small-integer columns, each either new or an exact integer combination of earlier ones (rank k/5)
* near_dependent: column k/2 is a combination of the earlier ones plus noise of delta times its norm, delta straddling
  the threshold 64 eps below which the Gram-Schmidt route replaces a column by a unit vector
* graded: singular values graded from 1 down to 1e-8, 1e-12, 1e-15
* zero_columns: zero column 0 (and a few more), trailing zero columns, the all-zero block
* unit_span: columns spanning e0 and e1 before a dependent column, so that the completion must skip those units; and
  range(A) = span(e0 .. e_{r-1}) with m - r dependent columns, so that square and wide blocks need every unit vector
* column_scale: columns scaled by powers of two from 2^-1050 to 2^1000 (their squares over- and underflow)

Bounds (eps = 2^-52, p = max(m, n), k = min(m, n), eta = 2^-1074 the spacing of the subnormal doubles), for every block:
* Q and R finite, R exactly upper triangular, diag(R) real and >= 0
* |Q^H Q - 1|_2 <= C p eps
* Gram-Schmidt, column by column: |(QR - A)_j| <= C p eps |a_j| + sqrt(k) m eta.  Independent of the scale of each column;
  the last term is the rounding of R = Q^T A to subnormal numbers, which matters only where a_j is itself subnormal
* Householder: |QR - A|_F <= C p eps |A|_F + sqrt(kn) eta
* a column j < k at distance d_j from the span of the columns before it: |R_jj - d_j| <= C p eps |a_j| (d_j = 0 for the
  exactly dependent and the zero columns)
* where the first r columns span range(A): |(1 - U_r U_r^H) Q_r|_2 <= C p eps kappa_r and |R_{r.., :}|_F <=
  C p eps kappa_r |A|_F, with U_r and kappa_r = s_1 / s_r from LAPACK's SVD.  Where a dependent column comes before an
  independent one, the vector Q has for it takes part in the later columns, and no unpivoted QR promises more than the
  previous item
* full-rank blocks with C p eps kappa <= 1e-3: Q and R equal LAPACK's factors (diag(R) made >= 0) to C p eps kappa for Q,
  and for R to that times |a_j| (Gram-Schmidt) or |A|_F (Householder).  kappa is the condition number of the first k
  columns after the scaling the route is invariant under: each column to max |a_ij| in [1, 2) for Gram-Schmidt, the whole
  block for Householder
Each test prints the largest measured ratio to each bound, per route.
"""
import numpy as np
import pytest

EPS = np.finfo(np.float64).eps
ETA = 2.**-1074
C = 4.
SHAPES = [(7, 5), (384, 384), (385, 385), (385, 3), (1000, 400), (3, 385), (300, 420)]


# ------------------------------------------------------------------ inputs: build(m, n, rs, rv) -> (A, meta)
# rs draws the structure (positions, coefficients, scales), rv the values: two draws with the same rs share the structure
def _int_combos(rs, B, n, ind):
    """m x n: column ind[t] is B[:, t], every other column an exact combination, with integer coefficients -2 .. 2, of
    the columns of `ind` before it (a zero column where there is none)"""
    r = B.shape[1]
    coef = np.zeros((r, n))
    t = 0
    for j in range(n):
        if t < r and ind[t] == j:
            coef[t, j] = 1.
            t += 1
        else:
            coef[:t, j] = rs.integers(-2, 3, t)
    return B @ coef


def _exact_rank(m, n, rs, rv, leading):
    k = min(m, n)
    r = k - 1 if k < 10 else k // 5
    ind = np.arange(r) if leading else np.sort(np.r_[0, rs.choice(np.arange(1, k), r - 1, replace=False)])
    B = rv.integers(-2, 3, (m, r)).astype(np.float64)
    assert np.linalg.matrix_rank(B) == r
    return _int_combos(rs, B, n, ind), dict(dep=sorted(set(range(k)) - set(ind)), rank=r if leading else None)


def _near_dependent(m, n, rs, rv, delta):
    j = min(m, n) // 2
    A = rv.standard_normal((m, n))
    b = A[:, :j] @ rs.standard_normal(j)
    u = rv.standard_normal(m)
    A[:, j] = b + delta * np.linalg.norm(b) / np.linalg.norm(u) * u
    return A, dict(near=j, full=True)


def _graded(m, n, rs, rv, g):
    k = min(m, n)
    U = np.linalg.qr(rv.standard_normal((m, k)))[0]
    V = np.linalg.qr(rs.standard_normal((n, k)))[0]
    return (U * np.logspace(0., np.log10(g), k)) @ V.T, dict(full=True)


def _zero_columns(m, n, rs, rv, where):
    k = min(m, n)
    A = rv.standard_normal((m, n))
    rank = None
    if where == 'all':
        z, rank = np.arange(n), 0
    elif where == 'trailing':
        z = np.arange(n - max(1, n // 8), n)
        rank = min(m, int(z[0]))
    else:
        z = np.r_[0, rs.choice(np.arange(1, n), max(1, n // 8), replace=False)]
    A[:, z] = 0.
    return A, dict(dep=[int(j) for j in z if j < k], rank=rank)


def _unit_span(m, n, rs, rv, kind):
    k = min(m, n)
    if kind == 'e0e1':
        # columns 0, 1 = e0 + e1, e0 - e1; column 2 depends on them: its completion has to skip e0 and e1
        ind = np.r_[0, 1, 3 + np.flatnonzero(rs.random(n - 3) < .75)]
        B = rv.integers(-2, 3, (m, len(ind))).astype(np.float64)
        B[:, :2] = 0.
        B[0, :2] = B[1, 0] = 1.
        B[1, 1] = -1.
        rank = None
    else:
        # range(A) = span(e0 .. e_{r-1}), every other column dependent: the completion skips r units and takes the
        # k - r after them -- for k = m every unit vector there is
        r = max(1, k // 2)
        B = np.zeros((m, r))
        B[:r] = rv.integers(-1, 2, (r, r))
        B[np.arange(r), np.arange(r)] = rv.choice([-4 * r, 4 * r], r)   # diagonally dominant, also made complex
        ind, rank = np.arange(r), r
    return _int_combos(rs, B, n, ind), dict(dep=sorted(set(range(k)) - set(ind)), rank=rank)


def _column_scale(m, n, rs, rv, _):
    e = rs.permutation(np.round(np.linspace(-1050, 1000, n)).astype(np.int64))
    return np.ldexp(rv.standard_normal((m, n)), e[None, :]), dict(full=True)


CLASSES = {
    'exact_rank': (_exact_rank, [True, False]),
    'near_dependent': (_near_dependent, [1e-6, 1e-10, 1e-13, 1e-14, 1e-15, 0.]),
    'graded': (_graded, [1e-8, 1e-12, 1e-15]),
    'zero_columns': (_zero_columns, ['first', 'trailing', 'all']),
    'unit_span': (_unit_span, ['e0e1', 'every_unit']),
    'column_scale': (_column_scale, [None]),
}


def _draw(name, variant, block, cplx):
    build, args = CLASSES[name]
    m, n = SHAPES[block]
    seed = [sorted(CLASSES).index(name), variant, block]

    def one(part):
        return build(m, n, np.random.default_rng(seed), np.random.default_rng(seed + [part]), args[variant])
    A, meta = one(1)
    if cplx:
        A = (1 + 2j) * A + 1j * one(2)[0]
    return A, meta


# ------------------------------------------------------------------ checks
def _ldexp(x, e):
    """x * 2^e, exact (no over- or underflow for the exponents used here)"""
    if np.iscomplexobj(x):
        return np.ldexp(x.real, e) + 1j * np.ldexp(x.imag, e)
    return np.ldexp(x, e)


def _exponent(x, axis=None):
    """e with max |x| * 2^e in [1, 2) (0 where x is zero), over `axis`"""
    mx = np.max(np.abs(x), axis=axis, initial=0.)
    return np.where(mx > 0., 1 - np.frexp(mx)[1], 0)


def _ratio(err, bound):
    """err / bound, elementwise; 0 / 0 = 0"""
    err, bound = np.broadcast_arrays(np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64))
    return np.max(np.where(bound > 0., err / np.where(bound > 0., bound, 1.), np.where(err > 0., np.inf, 0.)),
                  initial=0.)


def _record(stats, key, r):
    stats[key] = max(stats.get(key, 0.), float(r))
    assert r <= 1., (key, r)


def _check_block(A, Q, R, meta, route, stats):
    m, n = A.shape
    k, p = min(m, n), max(m, n)
    cplx = np.iscomplexobj(A)
    tag = route + ' '
    assert np.all(np.isfinite(Q)) and np.all(np.isfinite(R))
    assert np.all(np.tril(R, -1) == 0.)
    d = np.diag(R)
    assert np.all(d.imag == 0.)
    assert np.all(d.real >= 0.), ('diag(R) < 0', route, A.shape, float(d.real.min()))
    tol = C * p * EPS
    _record(stats, tag + 'orthogonality', _ratio(np.linalg.norm(Q.conj().T @ Q - np.eye(k), 2), tol))
    # reconstruction, on the scaled block (exact): column by column for Gram-Schmidt, normwise for Householder
    gs = route == 'gram-schmidt'
    e = _exponent(A, axis=0) if gs else np.full(n, _exponent(A))
    As, Rs = _ldexp(A, e[None, :]), _ldexp(R, e[None, :])
    under = np.ldexp(np.sqrt(k) * m * ETA if gs else np.sqrt(k * n) * ETA, e)      # eta term, scaled like the column
    col = np.linalg.norm(As, axis=0)
    if gs:
        _record(stats, tag + 'reconstruction', _ratio(np.linalg.norm(Q @ Rs - As, axis=0), tol * col + under))
    else:
        _record(stats, tag + 'reconstruction', _ratio(np.linalg.norm(Q @ Rs - As), tol * np.linalg.norm(As) + under[0]))
    # R_jj = distance of a_j from the span of the columns before it
    for j in meta.get('dep', []):
        _record(stats, tag + 'dependent R_jj', _ratio(abs(d[j]), tol * np.linalg.norm(A[:, j])))
    j = meta.get('near')
    if j is not None:
        x = np.linalg.lstsq(As[:, :j], As[:, j], rcond=None)[0]
        dist = np.linalg.norm(As[:, j] - As[:, :j] @ x)
        _record(stats, tag + 'near R_jj', _ratio(abs(Rs[j, j] - dist), tol * col[j]))
    # exact rank r with the first r columns spanning range(A): Q_r spans it, the rows of R below r vanish
    r = meta.get('rank')
    if r is not None:
        U, s, _ = np.linalg.svd(As, full_matrices=False)
        assert r == 0 or s[r - 1] > 1e3 * tol * s[0] and (r == k or s[r] <= tol * s[0]), 'test input: rank is not r'
        kap = s[0] / s[r - 1] if r else 1.
        Qr, Ur = Q[:, :r], U[:, :r]
        _record(stats, tag + 'span', _ratio(np.linalg.norm(Qr - Ur @ (Ur.conj().T @ Qr), 2) if r else 0., tol * kap))
        _record(stats, tag + 'rows below rank', _ratio(np.linalg.norm(Rs[r:]), tol * kap * np.linalg.norm(As)))
    # full rank and well conditioned: LAPACK's factors
    if meta.get('full'):
        s = np.linalg.svd(As[:, :k], compute_uv=False)
        kap = s[0] / s[-1] if s[-1] > 0. else np.inf
        if tol * kap <= 1e-3:
            QL, RL = np.linalg.qr(As)
            dl = np.diag(RL)
            ph = np.where(dl.real < 0., -1., 1.)
            if cplx:
                ph = dl / np.abs(dl)
            QL, RL = QL * ph[None, :], RL * ph.conj()[:, None]
            _record(stats, tag + 'Q = LAPACK', _ratio(np.max(np.abs(Q - QL)), tol * kap))
            ref = col if gs else np.full(n, np.linalg.norm(As))
            _record(stats, tag + 'R = LAPACK', _ratio(np.linalg.norm(Rs - RL, axis=0), tol * kap * ref + under))
            stats[tag + 'LAPACK compared'] = stats.get(tag + 'LAPACK compared', 0) + 1


def _check_class(name, cplx):
    from tenpy_b200.linalg import np_conserved as npc
    ci = npc.ChargeInfo([1], ['N'])
    rows = np.cumsum([0] + [s[0] for s in SHAPES])
    cols = np.cumsum([0] + [s[1] for s in SHAPES])
    charges = [[i] for i in range(len(SHAPES))]
    legs = [npc.LegCharge.from_qind(ci, rows, charges, +1), npc.LegCharge.from_qind(ci, cols, charges, -1)]
    qdata = [[i, i] for i in range(len(SHAPES))]
    big = [max(s) > npc.QR_HOUSEHOLDER_MAX for s in SHAPES]
    assert any(big) and not all(big)
    stats = {}
    for v in range(len(CLASSES[name][1])):
        blocks, metas = zip(*(_draw(name, v, b, cplx) for b in range(len(SHAPES))))
        a = npc.Array.from_blocks(legs, qdata, list(blocks), None, ['a', 'b'])
        assert np.dtype(a.dtype).kind == ('c' if cplx else 'f')
        n_cols = npc.qr_stats['columns']
        Q, R = npc.qr(a, inner_labels=['q', 'r'])
        # the route: the Gram-Schmidt columns are those of the real blocks above the cut-off
        assert npc.qr_stats['columns'] - n_cols == (0 if cplx else sum(min(s) for s, g in zip(SHAPES, big) if g))
        q, r = Q.to_ndarray(), R.to_ndarray()
        inner = Q.legs[1].slices
        for i, (A, meta) in enumerate(zip(blocks, metas)):
            route = 'complex householder' if cplx else 'gram-schmidt' if big[i] else 'householder'
            qb = q[rows[i]:rows[i + 1], inner[i]:inner[i + 1]]
            rb = r[inner[i]:inner[i + 1], cols[i]:cols[i + 1]]
            assert qb.shape == (A.shape[0], min(A.shape)) and rb.shape == (min(A.shape), A.shape[1])
            _check_block(A, qb, rb, meta, route, stats)
    print('\nnpc.qr %s %s: largest measured ratio to each bound' % (name, 'complex' if cplx else 'real'))
    for key in sorted(stats):
        print('  %-45s %.3g' % (key, stats[key]))


CASES = [pytest.param(name, cplx, id='%s-%s' % (name, 'complex' if cplx else 'real'))
         for name in CLASSES for cplx in (False, True)]


@pytest.mark.parametrize('name, cplx', CASES)
def test_qr_rank_deficient_host_logic(fake_device, name, cplx):
    _check_class(name, cplx)


@pytest.mark.gpu
@pytest.mark.parametrize('name, cplx', CASES)
def test_qr_rank_deficient_gpu(gpu_lib, name, cplx):
    _check_class(name, cplx)
