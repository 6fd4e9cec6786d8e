"""A real 4:2:0 JPEG transcode with LZ77-coded HF streams: tests/golden/genshin_ycbcr_420/input.jxl restreamed at test
time by tools/hf_restream.cc (rle and match), which rewrites only the HF pass codes, the pass groups' HF bits and the
TOC. The oracle must decode the restreamed file to the original's coefficients and pixels and reconstruct the original
JPEG from it; the host emulation of the subsampled LZ77 lanes variant must match the oracle, taking as many values from
copies as the restreamer wrote."""
import hashlib
import os
import sys

import numpy as np
import pytest

import jbr_lib
import oracle_lib
from test_hf_lz77 import _copied, emu  # noqa: F401  (emu: the counting emulation fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import hf_restream  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "genshin_ycbcr_420")


def original():
    with open(os.path.join(GOLDEN, "input.jxl"), "rb") as f:
        return f.read()


def jpeg_sha256():
    with open(os.path.join(GOLDEN, "ref_jpeg_sha256.txt")) as f:
        return f.read().split()[0]


_CACHE = {}


def restreamed(mode):
    if mode not in _CACHE:
        _CACHE[mode] = hf_restream.restream(original(), mode)
    return _CACHE[mode]


def _boxes(data):
    out, at = [], 0
    while at < len(data):
        n = int.from_bytes(data[at:at + 4], "big")
        out.append((data[at + 4:at + 8], data[at:at + n]))
        at += n
    return out


@pytest.mark.parametrize("mode", ["rle", "match"])
def test_only_the_hf_data_changes(mode):
    """Every box but the last codestream part is byte-identical, and that part starts as before."""
    data, copied = restreamed(mode)
    assert copied > 0 and data != original()
    a, b = _boxes(original()), _boxes(data)
    assert [t for t, _ in a] == [t for t, _ in b]
    assert b"jbrd" in [t for t, _ in a]
    for (_, x), (_, y) in zip(a[:-1], b[:-1]):
        assert x == y
    assert a[-1][1][8:20] == b[-1][1][8:20]  # the part index and the headers ahead of the TOC


@pytest.mark.parametrize("mode", ["rle", "match"])
def test_restreamed_file_decodes_like_the_original(mode):
    want = oracle_lib.OracleImage(original(), threads=8, capture=True)
    got = oracle_lib.OracleImage(restreamed(mode)[0], threads=8, capture=True)
    wc, gc = want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32)
    assert len(wc) == len(gc) == 3
    for w, g in zip(wc, gc):
        assert w.shape == g.shape and np.array_equal(w, g)
    assert np.array_equal(want.frame(0)[0].view(np.uint32), got.frame(0)[0].view(np.uint32))


@pytest.mark.parametrize("mode", ["rle", "match"])
def test_oracle_reconstructs_the_original_jpeg(mode):
    assert hashlib.sha256(jbr_lib.reconstruct_jpeg(restreamed(mode)[0])).hexdigest() == jpeg_sha256()


@pytest.mark.parametrize("mode", ["rle", "match"])
def test_emulated_lanes_match_oracle(emu, mode):  # noqa: F811
    data, copied = restreamed(mode)
    want = oracle_lib.OracleImage(data, threads=8, capture=True)
    before = _copied()
    got = oracle_lib.OracleImage(data, threads=8, capture=True, emu=True)
    assert _copied() - before == copied
    for w, g in zip(want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32)):
        assert np.array_equal(w, g)
    assert np.array_equal(want.frame(0)[0].view(np.uint32), got.frame(0)[0].view(np.uint32))
