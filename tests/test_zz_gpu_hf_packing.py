"""Streams per warp of the thread-per-stream HF coefficient kernel (jxlb_set_hf_streams_per_warp): every K with 64 and
128 streams per CTA, on each kernel variant the launcher can pick -- staged ANS, general (five HF presets' cluster maps
exceed the staging budget), LZ77, and chroma-subsampled (a JPEG transcode) -- against the oracle bit for bit, HF
coefficients and final planes; the 8K bench frame through the pipeline (default K); and corrupt streams, which must fail
with the same error class for every K."""
import ctypes
import subprocess

import numpy as np
import pytest

import bench
from conftest import fixture_bytes

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

KS = [4, 8, 16, 32]
PER_CTA = [64, 128]


def _lz77(tmp_path, mode):
    out = tmp_path / f"lz77_{mode}.jxl"
    subprocess.run([bench.synth_tool(), "--width", "1000", "--height", "600", "--seed", "7", "-o", str(out), "--hf-lz77", mode],
                   capture_output=True, text=True, check=True)
    return out.read_bytes()


FRAMES = {
    "staged": lambda tmp: bench.synth_frame(2000, 1500, 3, extra=("--passes", "2")),
    "general": lambda tmp: bench.synth_frame(1000, 600, 7, extra=("--hf-presets", "5", "--passes", "2")),
    "lz77_rle": lambda tmp: _lz77(tmp, "rle"),
    "lz77_match": lambda tmp: _lz77(tmp, "match"),
    "subsampled": lambda tmp: fixture_bytes("genshin_ycbcr_420", "input.jxl"),
}


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def want(oracle, tmp_path_factory):
    """Oracle planes and HF coefficients of each frame, computed once."""
    tmp = tmp_path_factory.mktemp("hf_packing")
    out = {}
    for name, make in FRAMES.items():
        data = make(tmp)
        img = oracle.OracleImage(data, threads=16, capture=True)
        out[name] = (data, img.frame(0)[0], img.stage("hf_coeff", np.int32))
        img.close()
    return out


def _schedule(dec, per_cta, k):
    dec.set_hf_streams_per_cta(per_cta)
    dec.set_hf_streams_per_warp(k)


def _reset(dec):
    dec.set_hf_streams_per_cta(0)
    dec.set_hf_streams_per_warp(0)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("per_cta", PER_CTA)
@pytest.mark.parametrize("frame", list(FRAMES))
def test_packing_matches_oracle(dec, want, frame, per_cta, k):
    data, planes, coeff = want[frame]
    _schedule(dec, per_cta, k)
    try:
        dec.set_capture(True)
        dec.decode(data)
        got = dec.frame_planar(0)
        gc = dec.stage("hf_coeff", np.int32)
        assert len(gc) == len(coeff) > 0
        for g, w in zip(gc, coeff):
            assert np.array_equal(g, w), "HF coefficient decode differs"
        assert got.shape == planes.shape
        assert np.array_equal(got.view(np.uint32), planes.view(np.uint32))
    finally:
        dec.set_capture(False)
        _reset(dec)


@pytest.fixture(scope="module")
def single_pass(oracle):
    data = bench.synth_frame(2000, 1500, 3)
    img = oracle.OracleImage(data, threads=16, capture=True)
    coeff = img.stage("hf_coeff", np.int32)
    img.close()
    return data, coeff


@pytest.mark.parametrize("k", KS)
def test_packing_decode_hf_groups(dec, single_pass, k):
    """jxlb_decode_hf_groups (HF coefficients into caller device planes), 128 streams per CTA."""
    data, coeff = single_pass
    _schedule(dec, 128, k)
    try:
        got = dec.decode_hf_groups(data)
        assert len(got) == len(coeff) == 3
        for g, w in zip(got, coeff):
            assert tuple(g.shape) == w.shape and np.array_equal(g.cpu().numpy(), w)
    finally:
        _reset(dec)


def _error_code(dec, data):
    import jxl_oxide_b200 as J
    try:
        dec.decode(data)
        return 0
    except J.JxlError as e:
        return e.code


@pytest.mark.parametrize("per_cta", PER_CTA)
def test_packing_corrupt_streams_fail_alike(dec, per_cta):
    """Bit flips in the HF sections and truncations: each K reports what K = 32 reports, and the decoder stays usable."""
    data = bench.synth_frame(1000, 600, 7)
    rng = np.random.default_rng(11)
    cases = [data[:len(data) // 2], data[:len(data) - 9]]
    for _ in range(10):
        m = bytearray(data)
        for pos in rng.integers(len(m) // 2, len(m), size=3):
            m[pos] ^= 1 << int(rng.integers(0, 8))
        cases.append(bytes(m))
    try:
        results = []
        for case in cases:
            codes = {}
            for k in (32, 16, 8, 4):
                _schedule(dec, per_cta, k)
                codes[k] = _error_code(dec, case)
            assert len(set(codes.values())) == 1, codes
            results.append(codes[32])
        assert results[1] != 0  # the stream cut short in its last HF section fails
        _schedule(dec, per_cta, 8)
        assert _error_code(dec, data) == 0
    finally:
        _reset(dec)


def _as_array(addr, nbytes, dtype, shape):
    buf = (ctypes.c_uint8 * nbytes).from_address(addr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()


def test_bench_frame_through_pipeline(oracle):
    """The 8K bench frame through the pipeline's thread-per-stream schedule at its default streams per warp."""
    import jxl_oxide_b200 as J
    data = bench.synth_frame(7680, 4320, 1)
    img = oracle.OracleImage(data, threads=32)
    w = img.frame(0)[0]
    img.close()
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for i in range(3):
            p.submit(data=data, mode=p.OUT_PLANAR_F32, tag=i)
        n = 0
        while p.in_flight:
            _, addr, nbytes = p.wait(want_output=True)
            assert nbytes == w.nbytes
            got = _as_array(addr, nbytes, np.float32, w.shape)
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint32), w.view(np.uint32))
            n += 1
        assert n == 3
    finally:
        p.close()
