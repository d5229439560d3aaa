"""FP64 products on the int8 tensor path (csrc/ozaki.cu): the splitting scheme emulated in numpy (CPU, documents and
pins the error model) and the CUDA kernels against a long-double product (gpu)."""
import numpy as np
import pytest


from fake_device import _FakeSplit, ozaki_product


def ozaki_emulated(A, B, slices):
    """(A B) by the scheme of csrc/ozaki.cu (numpy emulation in tests/fake_device.py: row-wise scaled signed 7-bit digits,
    exact integer slice products, diagonals summed in FP64 from the least significant pass)"""
    a, b = _FakeSplit(np.ascontiguousarray(A), slices), _FakeSplit(np.ascontiguousarray(B.T), slices)
    assert np.abs(a.digits).max() <= 64 and np.abs(b.digits).max() <= 64
    return ozaki_product(a, b)


def _cases(rng):
    A = rng.standard_normal((70, 150))
    B = rng.standard_normal((150, 90))
    yield 'gaussian', A, B
    U, _ = np.linalg.qr(rng.standard_normal((96, 96)))
    V, _ = np.linalg.qr(rng.standard_normal((96, 96)))
    yield 'theta-like', (U * np.logspace(0, -17, 96)) @ V, rng.standard_normal((96, 64))
    yield 'row-graded', A * np.logspace(0, -12, 70)[:, None], B * np.logspace(3, -9, 90)[None, :]
    A0 = A.copy()
    A0[5] = 0.
    yield 'zero row', A0, B


@pytest.mark.parametrize('slices,bound', [(6, 3e-11), (7, 3e-13), (8, 3e-15), (9, 1e-15)])
def test_ozaki_scheme_error_model(slices, bound):
    """error of the emulated scheme relative to the componentwise bound (|A||B|)_ij"""
    rng = np.random.default_rng(7)
    for name, A, B in _cases(rng):
        ref = (A.astype(np.longdouble) @ B.astype(np.longdouble))
        den = np.abs(A) @ np.abs(B) + 1e-300
        err = float(np.max(np.abs(ozaki_emulated(A, B, slices) - ref) / den))
        assert err < bound, (name, slices, err)


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(128, 128, 64), (70, 90, 150), (300, 260, 500), (129, 1, 17), (1, 300, 65),
                                   (513, 640, 1030)])
def test_ozaki_gemm_gpu(gpu_lib, shape):
    """b200_ozaki_split_f64 + b200_ozaki_mm_f64 against a long-double product and against the numpy emulation of the
    scheme (which the kernel must reproduce up to the FP64 summation order of the diagonals)"""
    import torch
    from tenpy_b200 import backend
    lib = gpu_lib
    m, n, k = shape
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    A = rng.standard_normal((m, k)) * np.logspace(0, -6, m)[:, None]
    B = rng.standard_normal((k, n)) * np.logspace(2, -3, n)[None, :]
    if m > 5:
        A[3] = 0.
    ref = (A.astype(np.longdouble) @ B.astype(np.longdouble))
    den = np.abs(A) @ np.abs(B) + 1e-300
    dA, dB = backend.to_device(A), backend.to_device(B)
    for slices, bound in ((7, 3e-13), (8, 3e-15), (4, 1e-5)):
        a_s = lib.ozaki_split(m, k, dA, k, 1, slices)
        b_s = lib.ozaki_split(n, k, dB, 1, n, slices)
        C = torch.full((m * n,), float('nan'), dtype=torch.float64, device=lib.device)
        lib.ozaki_mm(m, n, k, slices, a_s, b_s, C, n)
        lib.ozaki_check_abort()
        got = backend.to_host(C).reshape(m, n)
        assert np.all(np.isfinite(got))
        err = float(np.max(np.abs(got - ref) / den))
        assert err < bound, (shape, slices, err)
        emu = ozaki_emulated(A, B, slices)
        assert np.max(np.abs(got - emu) / den) < 1e-15, (shape, slices)
        # accumulate: C += A.B
        lib.ozaki_mm(m, n, k, slices, a_s, b_s, C, n, accumulate=True)
        got2 = backend.to_host(C).reshape(m, n)
        assert np.max(np.abs(got2 - 2 * got) / den) < 1e-15


@pytest.mark.gpu
def test_ozaki_gemm_strided_output_gpu(gpu_lib):
    """ldc > n (the product lands inside a wider packed buffer) and an operand reused across products"""
    import torch
    from tenpy_b200 import backend
    lib = gpu_lib
    rng = np.random.default_rng(3)
    m, n, k, ldc = 200, 150, 320, 190
    A, B1, B2 = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((k, n))
    a_s = lib.ozaki_split(m, k, backend.to_device(A), k, 1, 8)
    C = torch.zeros(m * ldc, dtype=torch.float64, device=lib.device)
    for B in (B1, B2):
        b_s = lib.ozaki_split(n, k, backend.to_device(B), 1, n, 8)
        lib.ozaki_mm(m, n, k, 8, a_s, b_s, C, ldc)
        got = backend.to_host(C).reshape(m, ldc)
        assert np.max(np.abs(got[:, :n] - A @ B)) < 1e-12
        assert np.all(got[:, n:] == 0.)
    lib.ozaki_check_abort()


def test_tensordot_int8_route_host_logic(fake_device, monkeypatch):
    """npc.tensordot sends single large block products to the int8 path (thresholds lowered here): operand offsets,
    `_out`, the cache of constant operands, and a whole DMRG run through it reproduce the golden energy"""
    import helpers as h
    from tenpy_b200.linalg import np_conserved as npc
    from tenpy_b200.models import TFIChain
    from tenpy_b200.networks.mps import MPS
    from tenpy_b200.algorithms import dmrg
    monkeypatch.setitem(npc.OZAKI, 'enabled', True)
    monkeypatch.setitem(npc.OZAKI, 'min_flops', 0.)
    monkeypatch.setitem(npc.OZAKI, 'min_dim', 2)
    rng = np.random.default_rng(5)
    a = npc.Array.from_ndarray_trivial(rng.standard_normal((6, 5, 7)), labels=['a', 'b', 'c'])
    b = npc.Array.from_ndarray_trivial(rng.standard_normal((7, 5, 4)), labels=['c*', 'b*', 'd'])
    b.legs[0], b.legs[1] = b.legs[0].conj(), b.legs[1].conj()
    n0 = fake_device.calls.get('ozaki_mm', 0)
    c = npc.tensordot(a, b, axes=[['c', 'b'], ['c*', 'b*']])
    assert fake_device.calls.get('ozaki_mm', 0) == n0 + 1
    ref = np.tensordot(a.to_ndarray(), b.to_ndarray(), axes=[[2, 1], [0, 1]])
    assert np.max(np.abs(c.to_ndarray() - ref)) < 1e-13
    a2 = a.transpose(['a', 'b', 'c'])
    a2._oz_const = True
    b2 = b.transpose(['b*', 'c*', 'd'])
    n_split = fake_device.calls.get('ozaki_split', 0)
    for _ in range(3):
        c2 = npc.tensordot(a2, b2, axes=[['b', 'c'], ['b*', 'c*']], _oz_slices=7)
    assert fake_device.calls.get('ozaki_split', 0) == n_split + 1 + 3          # a2 once, b2 every time
    assert np.max(np.abs(c2.to_ndarray() - ref)) < 1e-11
    g = h.load('dmrg.npz')
    M = TFIChain({'L': 20, 'J': 1., 'g': 1., 'conserve': None})
    psi = MPS.from_product_state(M.lat_sites, ['up'] * 20)
    n0 = fake_device.calls.get('ozaki_mm', 0)
    res = dmrg.run(psi, M, {'mixer': None, 'max_E_err': 1e-10, 'combine': True, 'matvec_order': 'split',
                            'trunc_params': {'chi_max': 50, 'svd_min': 1e-10}})
    assert fake_device.calls.get('ozaki_mm', 0) > n0
    assert abs(res['E'] - g['tfi_E']) < 1e-10 * abs(g['tfi_E'])
    assert np.max(np.abs(psi.entanglement_entropy() - g['tfi_S'])) < 1e-8


@pytest.mark.gpu
def test_tensordot_int8_route_gpu(gpu_lib, monkeypatch):
    """npc.tensordot through oz_gemm_kernel when the int8 route is switched on (off by default)"""
    from tenpy_b200.linalg import np_conserved as npc
    monkeypatch.setitem(npc.OZAKI, 'enabled', True)
    monkeypatch.setitem(npc.OZAKI, 'min_flops', 0.)
    monkeypatch.setitem(npc.OZAKI, 'min_dim', 2)
    rng = np.random.default_rng(11)
    a = npc.Array.from_ndarray_trivial(rng.standard_normal((130, 3, 70)), labels=['a', 'b', 'c'])
    b = npc.Array.from_ndarray_trivial(rng.standard_normal((70, 3, 90)), labels=['c*', 'b*', 'd'])
    b.legs[0], b.legs[1] = b.legs[0].conj(), b.legs[1].conj()
    n0 = npc.OZAKI['calls']
    c = npc.tensordot(a, b, axes=[['c', 'b'], ['c*', 'b*']])
    gpu_lib.ozaki_check_abort()
    assert npc.OZAKI['calls'] == n0 + 1
    ref = np.tensordot(a.to_ndarray(), b.to_ndarray(), axes=[[2, 1], [0, 1]])
    assert np.max(np.abs(c.to_ndarray() - ref)) < 1e-13 * np.max(np.abs(ref))
