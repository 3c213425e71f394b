"""pytest configuration: the ``gpu`` marker, import paths, and test-side stand-ins for the third-party
modules the reference's tests import (gpflow / tensorflow / oct2py -- none installable offline):
``tests/shims`` provides a gpflow config stub, a bare tensorflow stub and an ``oct2py`` whose
``Oct2Py().gp0/gp1/gp2/conlin/gSin/reward/pred`` execute the reference's own ``.m`` files (vendored, unmodified, under
``tests/reference_tests/Matlab Code``) with the MATLAB-subset interpreter ``oracle/mrun.py``.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
SHIMS = os.path.join(ROOT, "tests", "shims")
if SHIMS not in sys.path:
    sys.path.insert(0, SHIMS)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import pytest
    # the reference's own (unmodified) test files under tests/reference_tests/ need the device: mark them ``gpu``
    ref_dir = os.path.join(ROOT, "tests", "reference_tests")
    for item in items:
        if os.path.dirname(str(item.fspath)) == ref_dir:
            item.add_marker(pytest.mark.gpu)
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
