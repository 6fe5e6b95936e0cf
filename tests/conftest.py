import os
import sys

# The oracle's OpenMP threads must not spin while they wait: on a GPU box whose host cores are shared with other jobs a spinning team
# turns every parallel region into a scheduling lottery (one run of the N = 100 parity tests took ten minutes instead of one).
# Set before anything loads an OpenMP runtime.
os.environ.setdefault("OMP_WAIT_POLICY", "passive")
os.environ.setdefault("OMP_PROC_BIND", "false")

import numpy as np  # noqa: E402
import pytest  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the CUDA library and the oracle once per session (no-ops when up to date)."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "brusselator_golden.npz")))


@pytest.fixture(scope="session")
def po():
    from oracle import pyoracle
    return pyoracle


@pytest.fixture(scope="session")
def nls():
    import nonlinearsolve_jl_b200 as m
    return m


@pytest.fixture(scope="session")
def ctx(nls):
    """A library context on cuda:0; GPU tests only.  Raises (never falls back) when there is no device."""
    return nls.Context(0)
