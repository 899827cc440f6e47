import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def ctx():
    import sylph_b200
    c = sylph_b200.Context(0)
    yield c
    c.close()


SEED_MODES = {
    # defaults: CTA-tile kernel for ASCII device input; host inputs of syl_sketch_reads are packed to 2 bits by the
    # worker pool (warp kernel, packed variant) and shipped in tiny chunks (many chunks, every staging slot recycled)
    "default+packed-ingest": {"SYL_INGEST_CHUNK": "8192"},
    # warp-autonomous persistent kernel on ASCII input, fed ASCII from the host (1 byte per base over PCIe)
    "warp+ascii-ingest": {"SYL_SEED_IMPL": "warp", "SYL_HOST_INGEST": "ascii"},
    # CTA-tile kernel everywhere it can run
    "cta+ascii-ingest": {"SYL_HOST_INGEST": "ascii"},
}


@pytest.fixture(params=list(SEED_MODES))
def seed_mode(request, monkeypatch):
    """Run a test once per seeding / ingest implementation (the library reads these variables per call)."""
    for k in ("SYL_SEED_IMPL", "SYL_HOST_INGEST", "SYL_INGEST_CHUNK"):
        monkeypatch.delenv(k, raising=False)
    for k, v in SEED_MODES[request.param].items():
        monkeypatch.setenv(k, v)
    return request.param


@pytest.fixture(params=["device-driven", "synchronous"])
def contain_mode(request, monkeypatch):
    """syl_query / syl_profile: device-driven path (one host sync) and the synchronous two-pass path."""
    monkeypatch.delenv("SYL_CONTAIN_SYNC", raising=False)
    if request.param == "synchronous":
        monkeypatch.setenv("SYL_CONTAIN_SYNC", "1")
    return request.param
