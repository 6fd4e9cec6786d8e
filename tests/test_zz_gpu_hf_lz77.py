"""LZ77 in the HF coefficient streams on the device: the LZ77 variant of the thread-per-stream kernel
(decode_hf_lanes_kernel<SUB, false, true>, kernels/hf_lanes.cuh) against the oracle, on frames from
tools/synth_enc.cc --hf-lz77. Its per-stream logic is pinned on the CPU by tests/test_hf_lz77.py."""
import ctypes
import re
import subprocess

import numpy as np
import pytest

import bench

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

FRAMES = [((1000, 600), 7, ()), ((2600, 700), 5, ("--all-types",)), ((1000, 600), 5, ("--passes", "3")),
          ((1000, 600), 7, ("--hf-presets", "5"))]
FRAME_IDS = ["1000x600", "2600x700_all_types", "passes3", "presets5"]
# the device reports a stream it rejects as DEVICE_DECODE (6) where the host oracle says BITSTREAM (1)
NORM = {6: 1}


def _encode(tmp_path, size, seed, extra, mode):
    out = tmp_path / f"{mode}_{size[0]}x{size[1]}_{seed}{''.join(extra)}.jxl"
    r = subprocess.run([bench.synth_tool(), "--width", str(size[0]), "--height", str(size[1]), "--seed", str(seed),
                        "-o", str(out), "--hf-lz77", mode] + list(extra), capture_output=True, text=True, check=True)
    assert re.search(r"hf-lz77 \S+: [1-9]\d* values copied", r.stderr), r.stderr
    return out.read_bytes()


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


def _check(dec, oracle, data, streams):
    dec.set_hf_streams_per_cta(streams)
    try:
        dec.set_capture(True)
        dec.decode(data)
        got = dec.frame_planar(0)
        img = oracle.OracleImage(data, threads=8, capture=True)
        want = img.frame(0)[0]
        gc, wc = dec.stage("hf_coeff", np.int32), img.stage("hf_coeff", np.int32)
        assert len(gc) == len(wc) > 0
        for g, w in zip(gc, wc):
            assert np.array_equal(g, w), "HF coefficient decode differs"
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    finally:
        dec.set_capture(False)
        dec.set_hf_streams_per_cta(0)


@pytest.mark.parametrize("streams", [0, 4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("mode", ["rle", "match"])
@pytest.mark.parametrize("size,seed,extra", FRAMES, ids=FRAME_IDS)
def test_lz77_frames_match_oracle(dec, oracle, tmp_path, size, seed, extra, mode, streams):
    _check(dec, oracle, _encode(tmp_path, size, seed, extra, mode), streams)


@pytest.mark.parametrize("mode", ["rle", "match"])
def test_lz77_decode_hf_groups(oracle, tmp_path, mode):
    import jxl_oxide_b200 as J
    data = _encode(tmp_path, (2600, 700), 5, ("--all-types",), mode)
    img = oracle.OracleImage(data, threads=8, capture=True)
    want = img.stage("hf_coeff", np.int32)
    img.close()
    d = J.Decoder(0)
    try:
        coeff = d.decode_hf_groups(data)
        assert len(coeff) == 3
        for g, w in zip(coeff, want):
            assert tuple(g.shape) == w.shape and np.array_equal(g.cpu().numpy(), w)
    finally:
        d.close()


def _as_array(addr, nbytes, dtype, shape):
    buf = (ctypes.c_uint8 * nbytes).from_address(addr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()


def test_lz77_and_plain_frames_in_the_pipeline(oracle, tmp_path):
    """LZ77 and plain frames interleaved, an 8K LZ77 frame among them; plain frames decoded afterwards are still right."""
    import jxl_oxide_b200 as J
    lz = [_encode(tmp_path, (7680, 4320), 1, (), "match"), _encode(tmp_path, (1000, 600), 7, (), "rle"),
          _encode(tmp_path, (2600, 700), 5, ("--all-types",), "match"), _encode(tmp_path, (1000, 600), 5, ("--passes", "3"), "rle")]
    plain = [bench.synth_frame(1000, 600, 7), bench.synth_frame(2600, 700, 5, extra=("--all-types",)), bench.synth_frame(2000, 1500, 3)]
    datas = [lz[0], plain[0], lz[1], plain[1], lz[2], lz[3], plain[2]]
    want = []
    for d in datas:
        img = oracle.OracleImage(d, threads=32)
        want.append(img.frame(0)[0])
        img.close()
    p = J.Pipeline(0, workers=6, heavy_frames=2)
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
        for i, d in enumerate(plain):  # plain frames after the LZ77 ones
            p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=i)
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            w = want[datas.index(plain[tag])]
            got = _as_array(addr, nbytes, np.float32, w.shape)
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint32), w.view(np.uint32))
    finally:
        p.close()


@pytest.mark.parametrize("mode", ["bad-first", "bad-length"])
def test_invalid_lz77_streams_are_error_values(dec, oracle, tmp_path, mode):
    import jxl_oxide_b200 as J
    data = _encode(tmp_path, (1000, 600), 7, (), mode)
    with pytest.raises(oracle.OracleError) as e1:
        oracle.OracleImage(data, threads=2)
    for streams in (0, 64, 128):
        dec.set_hf_streams_per_cta(streams)
        try:
            with pytest.raises(J.JxlError) as e2:
                dec.decode(data)
        finally:
            dec.set_hf_streams_per_cta(0)
        assert NORM.get(e2.value.code, e2.value.code) == NORM.get(e1.value.code, e1.value.code) == 1
    good = bench.synth_frame(1000, 600, 7)  # the decoder stays usable
    dec.decode(good)
    img = oracle.OracleImage(good, threads=8)
    assert np.array_equal(dec.frame_planar(0).view(np.uint32), img.frame(0)[0].view(np.uint32))
