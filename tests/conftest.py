"""pytest configuration: the ``gpu`` marker and the fixtures selecting the device library.

* ``-m gpu`` tests run the real CUDA library on ``cuda:0`` (fixture ``gpu_lib``) -- these are the parity
  tests proper; they call through the C ABI and compare against ``oracle/`` and ``tests/golden``.
* ``-m "not gpu"`` tests cover the oracle against the golden vectors, the host logic and the C-ABI symbol
  table.  Host-logic tests use the ``fake_device`` fixture (a numpy TEST DOUBLE of the device library, see
  tests/fake_device.py); it is never used by a gpu test and never by the package itself.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


@pytest.fixture
def gpu_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tenpy_b200 import backend
    from tenpy_b200._lib import DeviceLib
    lib = backend._state['lib']
    if not isinstance(lib, DeviceLib):
        lib = backend.use_library(DeviceLib())
    return lib


@pytest.fixture
def fake_device():
    from tenpy_b200 import backend
    from fake_device import FakeDeviceLib
    import torch
    old = backend._state['lib']
    lib = backend.use_library(FakeDeviceLib())
    # poison uninitialised buffers: any element the host logic forgets to write shows up as NaN in the results
    old_empty = backend.empty
    backend.empty = lambda n: torch.full((int(n),), float('nan'), dtype=torch.float64)
    yield lib
    backend.empty = old_empty
    backend.use_library(old)
