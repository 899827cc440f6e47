"""Shared test helpers (FASTX reading with needletail's seq() semantics, flat buffers, seeding modes)."""
import gzip
import os

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(REPO, "tests", "golden", "data")


def read_fastx(path):
    """-> list of (header_line_without_marker, sequence_bytes). Line endings stripped, multi-line
    FASTA joined, no case/alphabet normalisation (needletail 0.5.1 seq()/id() semantics)."""
    op = gzip.open if open(path, "rb").read(2) == b"\x1f\x8b" else open
    with op(path, "rb") as f:
        data = f.read()
    recs = []
    if not data:
        return recs
    lines = data.split(b"\n")
    if data[:1] == b">":
        name, chunks = None, []
        for ln in lines:
            ln = ln.rstrip(b"\r")
            if ln[:1] == b">":
                if name is not None:
                    recs.append((name, b"".join(chunks)))
                name, chunks = ln[1:], []
            else:
                chunks.append(ln)
        if name is not None:
            recs.append((name, b"".join(chunks)))
    elif data[:1] == b"@":
        i = 0
        while i + 3 < len(lines) + 1 and i < len(lines):
            if not lines[i]:
                i += 1
                continue
            name = lines[i].rstrip(b"\r")[1:]
            seq = lines[i + 1].rstrip(b"\r")
            recs.append((name, seq))
            i += 4
    else:
        raise ValueError("not fasta/fastq: " + path)
    return recs


def flatten(seqs):
    """list of bytes -> (uint8 buffer, uint64 offsets[n+1])"""
    off = np.zeros(len(seqs) + 1, dtype=np.uint64)
    if seqs:
        off[1:] = np.cumsum([len(s) for s in seqs], dtype=np.uint64)
    buf = np.frombuffer(b"".join(seqs), dtype=np.uint8).copy() if seqs else np.zeros(0, dtype=np.uint8)
    return buf, off


SEED_MODES = {
    # defaults: ASCII device input through k_seed; host inputs of syl_sketch_reads are packed to 2 bits by the
    # worker pool (k_seed, packed variant) and shipped in tiny chunks (many chunks, every staging slot recycled)
    "default+packed-ingest": {"SYL_INGEST_CHUNK": "8192"},
    # host inputs fed as ASCII (1 byte per base over PCIe); genome sketches through the generic radix-sort post-pass
    # instead of the slotted one.  The id is that of the former warp-kernel mode, so test ids stay stable.
    "warp+ascii-ingest": {"SYL_HOST_INGEST": "ascii", "SYL_GENOME_POSTPASS": "sort"},
    # ASCII everywhere, default post-passes
    "cta+ascii-ingest": {"SYL_HOST_INGEST": "ascii"},
}


@pytest.fixture(params=list(SEED_MODES))
def seed_mode(request, monkeypatch):
    """Run a test once per seeding input / post-pass mode (the library reads these variables per call)."""
    for k in ("SYL_HOST_INGEST", "SYL_INGEST_CHUNK", "SYL_GENOME_POSTPASS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in SEED_MODES[request.param].items():
        monkeypatch.setenv(k, v)
    return request.param
