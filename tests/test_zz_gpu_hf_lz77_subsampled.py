"""LZ77 in the HF coefficient streams of chroma-subsampled frames on the device: the subsampled LZ77 variant of the
thread-per-stream kernel (decode_hf_lanes_kernel<true, false, true>, kernels/hf_lanes.cuh) against the oracle, on frames
from tools/synth_enc.cc --ycbcr --hf-lz77 and on the 4:2:0 JPEG transcode tests/golden/genshin_ycbcr_420 restreamed with
LZ77 codes (tools/hf_restream.cc). Its per-stream logic is pinned on the CPU by tests/test_hf_lz77_subsampled.py and
tests/test_hf_lz77_restream.py. Every LZ77 code runs one schedule (128 streams per CTA, hf_schedule), whatever
hf_streams_per_cta says, so the tests do not vary it."""
import ctypes
import hashlib
import re
import subprocess

import numpy as np
import pytest

import bench
from test_hf_lz77_restream import jpeg_sha256, original, restreamed

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

FRAMES = [("420", (1, 1), 1), ("420", (257, 129), 2), ("422", (1000, 600), 1), ("440", (1000, 600), 2),
          ("420", (2600, 700), 1), ("444", (257, 129), 1)]
FRAME_IDS = [f"{m}_{s[0]}x{s[1]}_p{p}" for m, s, p in FRAMES]
# the device reports a stream it rejects as DEVICE_DECODE (6) where the host oracle says BITSTREAM (1)
NORM = {6: 1}


def _encode(tmp_path, mode, size, passes, lz, seed=3):
    out = tmp_path / f"{mode}_{size[0]}x{size[1]}_p{passes}_{lz}.jxl"
    r = subprocess.run([bench.synth_tool(), "--width", str(size[0]), "--height", str(size[1]), "--seed", str(seed),
                        "--ycbcr", mode, "--passes", str(passes), "-o", str(out), "--hf-lz77", lz],
                       capture_output=True, text=True, check=True)
    assert re.search(r"hf-lz77 \S+: \d+ values copied", r.stderr), r.stderr
    return out.read_bytes()


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


def _want(oracle, data):
    img = oracle.OracleImage(data, threads=8, capture=True)
    return img.frame(0)[0], img.stage("hf_coeff", np.int32)


def _same(got, want):
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def _check_decode(dec, oracle, data):
    want_px, want_coeff = _want(oracle, data)
    try:
        dec.set_capture(True)
        dec.decode(data)
        got = dec.stage("hf_coeff", np.int32)
        assert len(got) == len(want_coeff) == 3
        for g, w in zip(got, want_coeff):
            _same(g, w)
        _same(dec.frame_planar(0), want_px)
    finally:
        dec.set_capture(False)


@pytest.mark.parametrize("lz", ["rle", "match"])
@pytest.mark.parametrize("mode,size,passes", FRAMES, ids=FRAME_IDS)
def test_decode_matches_oracle(dec, oracle, tmp_path, mode, size, passes, lz):
    _check_decode(dec, oracle, _encode(tmp_path, mode, size, passes, lz))


@pytest.mark.parametrize("lz", ["rle", "match"])
def test_restreamed_transcode_decodes_like_oracle(dec, oracle, lz):
    _check_decode(dec, oracle, restreamed(lz)[0])


def _check_hf_groups(dec, oracle, data):
    """jxlb_decode_hf_groups into caller planes as wide as the full-resolution channel (the reported width is that of
    the first, subsampled one)."""
    import torch
    _, want = _want(oracle, data)
    h = max(p.shape[0] for p in want)
    w = max(p.shape[1] for p in want)
    planes = [torch.full((h, w), -7, dtype=torch.int32, device="cuda:0") for _ in range(3)]
    ptrs = (ctypes.c_void_p * 3)(*[int(p.data_ptr()) for p in planes])
    ow, oh = ctypes.c_uint32(), ctypes.c_uint32()
    dec._check(dec._L.jxlb_decode_hf_groups(dec._h, data, len(data), ptrs, w, ctypes.byref(ow), ctypes.byref(oh)))
    torch.cuda.synchronize()
    assert (ow.value, oh.value) == (want[0].shape[1], want[0].shape[0])
    for g, wp in zip(planes, want):
        _same(g.cpu().numpy()[:wp.shape[0], :wp.shape[1]], wp)


@pytest.mark.parametrize("lz", ["rle", "match"])
@pytest.mark.parametrize("mode,size,passes", FRAMES, ids=FRAME_IDS)
def test_decode_hf_groups(dec, oracle, tmp_path, mode, size, passes, lz):
    _check_hf_groups(dec, oracle, _encode(tmp_path, mode, size, passes, lz))


@pytest.mark.parametrize("lz", ["rle", "match"])
def test_restreamed_transcode_hf_groups(dec, oracle, lz):
    _check_hf_groups(dec, oracle, restreamed(lz)[0])


@pytest.mark.parametrize("lz", ["rle", "match"])
def test_restreamed_transcode_reconstructs_the_jpeg(dec, lz):
    """jxlb_reconstruct_jpeg and JxlImage.reconstruct_jpeg(): coefficients from the subsampled LZ77 lanes variant,
    scans encoded on the GPU."""
    import jxl_oxide_b200 as J
    data = restreamed(lz)[0]
    assert hashlib.sha256(dec.reconstruct_jpeg(data)).hexdigest() == jpeg_sha256()
    assert hashlib.sha256(J.JxlImage.read(data).reconstruct_jpeg()).hexdigest() == jpeg_sha256()


@pytest.mark.parametrize("which", FRAME_IDS[1:4] + ["restreamed_rle", "restreamed_match"])
def test_decode_keyframe(oracle, tmp_path, which):
    import jxl_oxide_b200 as J
    if which.startswith("restreamed_"):
        data = restreamed(which.split("_")[1])[0]
    else:
        mode, size, passes = FRAMES[FRAME_IDS.index(which)]
        data = _encode(tmp_path, mode, size, passes, "match")
    want, _ = _want(oracle, data)
    d = J.Decoder(0)
    try:
        d.decode_keyframe(data, 0)
        _same(d.frame_planar(0), want)
    finally:
        d.close()


def _as_array(addr, nbytes, dtype, shape):
    buf = (ctypes.c_uint8 * nbytes).from_address(addr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()


def test_pipeline(oracle, tmp_path):
    """Subsampled LZ77 frames, a subsampled plain frame and an XYB LZ77 frame interleaved in the pipeline."""
    import jxl_oxide_b200 as J
    datas = [_encode(tmp_path, m, s, p, lz) for (m, s, p), lz in zip(FRAMES, ["match", "rle", "match", "rle", "match", "rle"])]
    datas.append(bench.synth_frame(1000, 600, 3, extra=("--ycbcr", "420")))
    datas.append(bench.synth_frame(1000, 600, 7, extra=("--hf-lz77", "match")))
    datas += [restreamed("rle")[0], original(), restreamed("match")[0]]
    want = [_want(oracle, d)[0] for d in datas]
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for rep in range(2):
            for i, d in enumerate(datas):
                p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=100 * rep + i)
        seen = set()
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            w = want[tag % 100]
            assert nbytes == w.nbytes
            got = _as_array(addr, nbytes, np.float32, w.shape)
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint32), w.view(np.uint32)), f"frame {tag} differs from the oracle"
            seen.add(tag)
        assert len(seen) == 2 * len(datas)
    finally:
        p.close()


@pytest.mark.parametrize("bad", ["bad-first", "bad-length"])
@pytest.mark.parametrize("mode", ["420", "422", "440"])
def test_invalid_streams_are_error_values(dec, oracle, tmp_path, mode, bad):
    import jxl_oxide_b200 as J
    data = _encode(tmp_path, mode, (1000, 600), 1, bad)
    with pytest.raises(oracle.OracleError) as e1:
        oracle.OracleImage(data, threads=2)
    with pytest.raises(J.JxlError) as e2:
        dec.decode(data)
    assert NORM.get(e2.value.code, e2.value.code) == NORM.get(e1.value.code, e1.value.code) == 1
    good = _encode(tmp_path, mode, (1000, 600), 1, "rle")  # the decoder stays usable
    dec.decode(good)
    _same(dec.frame_planar(0), _want(oracle, good)[0])
