"""Host run of the Householder QR phases (tests/csrc/block_qr_host.cpp): the phases of block_qr_core.cuh executed for
every thread index exactly as block_qr_kernel executes them, compiled with the host C++ compiler, for real and for
complex blocks.  Checks QR = A, orthonormal Q and triangular R with a real non-negative diagonal at edge shapes, and
exact power-of-two equivariance of Q and R for 2^e A with |e| <= 990.  No GPU needed; skipped where no C++ compiler is
installed."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_block_qr_host_phases(tmp_path):
    cxx = next((c for c in (os.environ.get('CXX'), 'c++', 'g++', 'clang++') if c and shutil.which(c)), None)
    if cxx is None:
        pytest.skip('no host C++ compiler')
    exe = str(tmp_path / 'block_qr_host')
    subprocess.run([cxx, '-O2', '-std=c++17', '-o', exe, os.path.join(ROOT, 'tests', 'csrc', 'block_qr_host.cpp')],
                   check=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = res.stdout.splitlines()
    assert 'scale cases: ok' in lines
    assert 'complex scale cases: ok' in lines
    assert lines[-1] == 'ok'
