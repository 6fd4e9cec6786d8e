"""LZ77 in the HF coefficient streams of chroma-subsampled VarDCT frames (tools/synth_enc.cc --ycbcr with --hf-lz77).

`--ycbcr` writes a VarDCT frame laid out like a JPEG transcode (Cb, Y, Cr with jpeg_upsampling, DCT8 in every cell, no
chroma from luma, each channel's LF and HF at its shifted grid), and `--dump-coeffs` the coefficients it coded. The plain
frame is pinned on its own against that dump; the LZ77 frames must then give the oracle the same coefficients and pixels.
The host emulation of the thread-per-stream kernel (built with the copied-values count, tests/emu/hf_lz77.mk) runs the
device's subsampled LZ77 variant and must match the oracle bit for bit, with as many values copied as the encoder wrote.
"""
import random
import re
import subprocess

import numpy as np
import pytest

import bench
import oracle_lib
from test_hf_lz77 import _copied, _error_code, emu  # noqa: F401  (emu: the counting emulation fixture)

# (channel hshift, vshift) of Cb, Y, Cr per mode (ChannelShift::from_jpeg_upsampling)
SHIFTS = {"444": ((0, 0), (0, 0), (0, 0)), "420": ((1, 1), (0, 0), (1, 1)),
          "422": ((1, 0), (0, 0), (1, 0)), "440": ((0, 1), (0, 0), (0, 1))}
MODES = list(SHIFTS)
# 1x1, partial edge groups with odd sizes in the subsampled directions, several groups, more than one LF group
SIZES = [(1, 1), (257, 129), (1000, 600), (2600, 700)]
SIZE_IDS = ["1x1", "257x129", "1000x600", "2600x700"]
# LZ77 frames: every mode at the three smaller sizes, and two LF groups' worth of 4:2:0
LZ_CASES = [(m, s, p) for m in MODES for s in SIZES[:3] for p in (1, 2)] + [("420", (2600, 700), 1), ("420", (2600, 700), 2)]
LZ_IDS = [f"{m}_{s[0]}x{s[1]}_p{p}" for m, s, p in LZ_CASES]


def _encode(tmp_path, size, mode, passes, lz=None, seed=3):
    """(frame bytes, dumped coefficient planes, values copied as the encoder counted them)."""
    tag = f"{mode}_{size[0]}x{size[1]}_p{passes}_{lz or 'plain'}"
    out, dump = tmp_path / f"{tag}.jxl", tmp_path / f"{tag}.coeffs"
    args = [bench.synth_tool(), "--width", str(size[0]), "--height", str(size[1]), "--seed", str(seed), "--ycbcr", mode,
            "--passes", str(passes), "-o", str(out), "--dump-coeffs", str(dump)]
    if lz:
        args += ["--hf-lz77", lz]
    r = subprocess.run(args, capture_output=True, text=True, check=True)
    copied = None
    if lz:
        m = re.search(r"hf-lz77 \S+: (\d+) values copied", r.stderr)
        assert m, r.stderr
        copied = int(m.group(1))
    return out.read_bytes(), _planes(np.fromfile(dump, dtype=np.int32), size, mode), copied


def _planes(raw, size, mode):
    """The dump cut into the three channel planes (X / Cb, Y, B / Cr), each (blocks >> shift) * 8 samples a side."""
    hsub, vsub = mode in ("420", "422"), mode in ("420", "440")
    bw, bh = (size[0] + 7) // 8, (size[1] + 7) // 8
    bw, bh = (bw + 1) // 2 * 2 if hsub else bw, (bh + 1) // 2 * 2 if vsub else bh
    planes, off = [], 0
    for hs, vs in SHIFTS[mode]:
        w, h = (bw >> hs) * 8, (bh >> vs) * 8
        planes.append(raw[off:off + w * h].reshape(h, w))
        off += w * h
    assert off == raw.size
    return planes


def _same_coeffs(want, got):
    assert len(want) == len(got) == 3
    for w, g in zip(want, got):
        assert w.shape == g.shape and np.array_equal(w, g)


def _same_image(want, got):
    _same_coeffs(want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32))
    assert np.array_equal(want.frame(0)[0].view(np.uint32), got.frame(0)[0].view(np.uint32))


@pytest.mark.parametrize("passes", [1, 2])
@pytest.mark.parametrize("size", SIZES, ids=SIZE_IDS)
@pytest.mark.parametrize("mode", MODES)
def test_plain_frame_decodes_to_the_dumped_coefficients(tmp_path, mode, size, passes):
    data, coeffs, _ = _encode(tmp_path, size, mode, passes)
    img = oracle_lib.OracleImage(data, threads=4, capture=True)
    _same_coeffs(coeffs, img.stage("hf_coeff", np.int32))
    assert any(np.any(c) for c in coeffs)
    px = img.frame(0)[0]
    assert px.shape[1:] == (size[1], size[0]) and np.all(np.isfinite(px))


@pytest.mark.parametrize("lz", ["rle", "match"])
@pytest.mark.parametrize("mode,size,passes", LZ_CASES, ids=LZ_IDS)
def test_lz77_frame_decodes_like_plain_frame(tmp_path, mode, size, passes, lz):
    plain, coeffs, _ = _encode(tmp_path, size, mode, passes)
    data, coeffs_lz, copied = _encode(tmp_path, size, mode, passes, lz)
    assert data != plain
    if size != (1, 1):
        assert copied > 0
    _same_coeffs(coeffs, coeffs_lz)
    _same_image(oracle_lib.OracleImage(plain, threads=4, capture=True), oracle_lib.OracleImage(data, threads=4, capture=True))


@pytest.mark.parametrize("lz", ["rle", "match"])
@pytest.mark.parametrize("mode,size,passes", LZ_CASES, ids=LZ_IDS)
def test_emulated_subsampled_lz77_lanes_match_oracle(emu, tmp_path, mode, size, passes, lz):  # noqa: F811
    data, _, copied = _encode(tmp_path, size, mode, passes, lz)
    want = oracle_lib.OracleImage(data, threads=4, capture=True)
    before = _copied()
    got = oracle_lib.OracleImage(data, threads=4, capture=True, emu=True)
    assert _copied() - before == copied
    _same_image(want, got)


@pytest.mark.parametrize("bad", ["bad-first", "bad-length"])
@pytest.mark.parametrize("mode", ["420", "422", "440"])
def test_invalid_streams_give_the_oracles_error_class(emu, tmp_path, mode, bad):  # noqa: F811
    data, _, _ = _encode(tmp_path, (1000, 600), mode, 1, bad)
    want, _ = _error_code(data, emu=False)
    got, _ = _error_code(data, emu=True)
    assert want == 1 and got == want


@pytest.mark.parametrize("mode", ["420", "422"])
def test_mutated_frames_give_the_oracles_result(emu, tmp_path, mode):  # noqa: F811
    """Seeded byte mutations in the HF sections of a subsampled `match` frame: the emulation decodes to the oracle's
    pixels or fails with the oracle's error class."""
    data, _, _ = _encode(tmp_path, (1000, 600), mode, 1, "match")
    hf_start = len(data) // 3  # past LfGlobal, the LF group and HfGlobal: the HF sections hold most of the frame
    rng = random.Random(23)
    for _ in range(24):
        m = bytearray(data)
        for _ in range(rng.choice((1, 1, 2, 4))):
            m[rng.randrange(hf_start, len(m))] = rng.randrange(256)
        want, want_px = _error_code(bytes(m), emu=False)
        got, got_px = _error_code(bytes(m), emu=True)
        assert got == want
        if want_px is not None:
            assert np.array_equal(want_px.view(np.uint32), got_px.view(np.uint32))
