"""The doublecomplex path (pzgstrf3d_b200, SURVEY 8a row a15), the pzdrive3d drop-in and the overlapped upload: gating.
Each group runs in a child process (tests/optin_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(what):
    r = subprocess.run([sys.executable, os.path.join(HERE, "optin_worker.py"), what], capture_output=True, text=True,
                       timeout=420)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])


def test_optin_complex_kernels():
    _run("zkernels")


def test_optin_pzgstrf3d():
    _run("zfactor")


def test_optin_pzdrive3d_dropin():
    _run("zdropin")


def test_optin_overlapped_upload():
    _run("h2d")
