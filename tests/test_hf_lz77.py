"""LZ77 in the HF coefficient streams of VarDCT frames (tools/synth_enc.cc --hf-lz77).

An LZ77 frame and the plain frame of the same size, seed and flags carry the same coefficients, so the oracle must
decode both to identical HF coefficients and pixels: the plain path is pinned by the rest of the suite, so this checks
the host LZ77 reader and the encoder without trusting either alone. The host emulation of the thread-per-stream kernel
(tests/emu/, built by hf_lz77.mk with a count of copied values) then runs the device's LZ77 variant on the same frames,
and must match the oracle bit for bit, with as many values taken from copies as the encoder wrote.
"""
import ctypes
import os
import random
import re
import subprocess

import numpy as np
import pytest

import bench
import oracle_lib

FRAMES = [((1000, 600), 7, ()), ((1000, 600), 7, ("--all-types",)), ((2600, 700), 5, ("--all-types",)),
          ((1000, 600), 7, ("--passes", "2")), ((1000, 600), 5, ("--passes", "3")), ((1000, 600), 7, ("--hf-presets", "5")),
          ((2600, 700), 5, ("--all-types", "--passes", "2"))]
FRAME_IDS = ["1000x600", "1000x600_all_types", "2600x700_all_types", "passes2", "passes3", "presets5",
             "2600x700_all_types_passes2"]
# the device reports a stream it rejects as DEVICE_DECODE (6) where the host oracle says BITSTREAM (1)
NORM = {6: 1}


EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_LZ77_LIB = None


def _lz77_emu_lib():
    """The HF lanes emulation built with the count of values taken from LZ77 copies (tests/emu/hf_lz77.mk)."""
    global _LZ77_LIB
    if _LZ77_LIB is None:
        subprocess.check_call(["make", "-s", "-C", EMU, "-f", "hf_lz77.mk"])
        _LZ77_LIB = oracle_lib._load(os.path.join(EMU, "_build", "libjxlemu_lz77.so"), None)
        _LZ77_LIB.jxle_hf_lz77_copied.restype = ctypes.c_uint64
        _LZ77_LIB.jxle_hf_lz77_window_entries.restype = ctypes.c_uint64
        _LZ77_LIB.jxle_hf_lz77_window_entries.argtypes = [ctypes.c_uint32]
    return _LZ77_LIB


@pytest.fixture
def emu(monkeypatch):
    """OracleImage(..., emu=True) decodes with the counting build of the emulation."""
    monkeypatch.setattr(oracle_lib, "emu_lib", _lz77_emu_lib)


def _encode(tmp_path, size, seed, extra, mode):
    """(frame bytes, values the decoder takes from copies as the encoder counted them)."""
    out = tmp_path / f"{mode}_{size[0]}x{size[1]}_{seed}.jxl"
    r = subprocess.run([bench.synth_tool(), "--width", str(size[0]), "--height", str(size[1]), "--seed", str(seed),
                        "-o", str(out), "--hf-lz77", mode] + list(extra), capture_output=True, text=True, check=True)
    m = re.search(r"hf-lz77 \S+: (\d+) values copied, (\d+) copies from the first value", r.stderr)
    assert m, r.stderr
    return out.read_bytes(), int(m.group(1)), int(m.group(2))


def _copied():
    return _lz77_emu_lib().jxle_hf_lz77_copied()


def _assert_same(want, got):
    assert got.num_frames == want.num_frames
    for i in range(want.num_frames):
        assert np.array_equal(want.frame(i)[0].view(np.uint32), got.frame(i)[0].view(np.uint32)), f"frame {i} differs"
    ca, cb = want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32)
    assert len(ca) == len(cb) > 0
    for x, y in zip(ca, cb):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("mode", ["rle", "match"])
@pytest.mark.parametrize("size,seed,extra", FRAMES, ids=FRAME_IDS)
def test_lz77_frame_decodes_like_plain_frame(tmp_path, size, seed, extra, mode):
    data, copied, from_start = _encode(tmp_path, size, seed, extra, mode)
    plain = bench.synth_frame(size[0], size[1], seed, extra=extra)
    assert data != plain and copied > 0
    if mode == "match":
        assert from_start > 0  # distances beyond the values decoded so far, clamped by the decoder
    want = oracle_lib.OracleImage(plain, threads=4, capture=True)
    got = oracle_lib.OracleImage(data, threads=4, capture=True)
    _assert_same(want, got)


@pytest.mark.parametrize("mode", ["rle", "match"])
@pytest.mark.parametrize("size,seed,extra", FRAMES, ids=FRAME_IDS)
def test_emulated_lz77_lanes_match_oracle(emu, tmp_path, size, seed, extra, mode):
    data, copied, _ = _encode(tmp_path, size, seed, extra, mode)
    want = oracle_lib.OracleImage(data, threads=4, capture=True)
    before = _copied()
    got = oracle_lib.OracleImage(data, threads=4, capture=True, emu=True)
    assert _copied() - before == copied > 0
    _assert_same(want, got)


def _error_code(data, emu):
    try:
        img = oracle_lib.OracleImage(data, threads=2, emu=emu)
        px = img.frame(0)[0] if img.num_frames else None
        img.close()
        return None, px
    except oracle_lib.OracleError as e:
        return NORM.get(e.code, e.code), None


@pytest.mark.parametrize("mode", ["bad-first", "bad-length"])
def test_invalid_lz77_streams_give_the_oracles_error_class(emu, tmp_path, mode):
    data, _, _ = _encode(tmp_path, (1000, 600), 7, (), mode)
    want, _ = _error_code(data, emu=False)
    got, _ = _error_code(data, emu=True)
    assert want == 1 and got == want


def test_mutated_lz77_frames_give_the_oracles_result(emu, tmp_path):
    """Seeded byte mutations inside the HF sections of a `match` frame: the emulation decodes to the oracle's pixels or
    fails with the oracle's error class (a window index outside the window would abort the process)."""
    data, _, _ = _encode(tmp_path, (1000, 600), 7, (), "match")
    plain = bench.synth_frame(1000, 600, 7)
    hf_start = len(data) - 55000  # the HF sections take the last ~55 KB of the plain frame's 74 KB, more here
    assert len(plain) > 55000 and hf_start > 0
    rng = random.Random(11)
    for _ in range(36):
        m = bytearray(data)
        for _ in range(rng.choice((1, 1, 2, 4))):
            m[rng.randrange(hf_start, len(m))] = rng.randrange(256)
        want, want_px = _error_code(bytes(m), emu=False)
        got, got_px = _error_code(bytes(m), emu=True)
        assert got == want
        if want_px is not None:
            assert np.array_equal(want_px.view(np.uint32), got_px.view(np.uint32))


def test_window_size_per_group_dim():
    L = _lz77_emu_lib()
    assert [L.jxle_hf_lz77_window_entries(d) for d in (128, 256, 512, 1024)] == [49152, 196608, 786432, 1 << 20]
