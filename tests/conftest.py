"""pytest configuration: registers the `gpu` marker and puts the package + repo root on sys.path."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "open-sora_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu")


import pytest


@pytest.fixture
def fake_osb(monkeypatch):
    """Install the CPU stand-in of the binding (tests/fake_osb200.py) as `osb200` for one test: the host-side models
    import the binding lazily at call time, so their shape / stride / caching logic runs on the CPU against the
    documented contract of every entry point.  The real module is restored afterwards."""
    from tests import fake_osb200

    fake_osb200.reset()
    monkeypatch.setitem(sys.modules, "osb200", fake_osb200)
    return fake_osb200
