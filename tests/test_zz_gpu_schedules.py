"""GPU parity of the opt-in schedules and delivery paths: the thread-per-stream HF coefficient kernel
(decode_hf_lanes_kernel, kernels/hf_lanes.cuh) and packing into a device buffer (jxlb_frame_write_to_device).

The kernel is an opt-in schedule (jxlb_set_hf_streams_per_cta / JXLB_HF_LANES) of the same streams the default
one-warp-per-stream kernel decodes; its per-stream logic is pinned on the CPU by tests/test_emu_lanes.py. Here the
device launch is compared with the oracle (coefficients bit-identical, final pixels 0 ULP) and with the default
kernel's error behaviour. The file sorts last on purpose: it exercises an alternative schedule, after the product
defaults have been checked.
"""
import numpy as np
import pytest

import bench
from conftest import fixture_bytes

# These kernels / paths had not run on a GPU when the tests were written: if one of them ever blocks, end the run (this
# file sorts last, every other result is already out) instead of sitting in a blocked CUDA call until the box times out.
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]

FIXTURES = ["opsin_inverse", "bike", "cafe", "issue_425", "genshin_ycbcr_420", "bench_oriented_brg", "minecraft_vardct_e7", "upsampling"]
# streams per CTA: 8 and 32 run one warp per stream with every preset's tables staged once per CTA (decode_hf_warp_kernel;
# the default 16 runs in every other GPU test), 64 one thread per stream (decode_hf_lanes_kernel)
SCHEDULES = [8, 32, 64]


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
        for g, w in zip(dec.stage("hf_coeff", np.int32), img.stage("hf_coeff", np.int32)):
            assert np.array_equal(g, w), "HF coefficient decode differs"
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    finally:
        dec.set_capture(False)
        dec.set_hf_streams_per_cta(0)


@pytest.mark.parametrize("streams", SCHEDULES)
@pytest.mark.parametrize("name", FIXTURES)
def test_hf_lanes_fixture(dec, oracle, name, streams):
    _check(dec, oracle, fixture_bytes(name, "input.jxl"), streams)


@pytest.mark.parametrize("streams", [4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("extra", [(), ("--passes", "3")])
def test_hf_lanes_synthetic(dec, oracle, streams, extra):
    # 2000x1500: 8x6 groups (ragged right / bottom), more streams than one CTA carries at 32 per CTA
    _check(dec, oracle, bench.synth_frame(2000, 1500, 3, extra=extra), streams)


def test_hf_lanes_bench_file(dec, oracle):
    _check(dec, oracle, fixture_bytes("benchmark-data", "starrail.d1-e6.jxl"), 32)


def test_hf_lanes_errors_are_values(dec):
    import jxl_oxide_b200
    data = bytearray(bench.synth_frame(1000, 600, 7))
    rng = np.random.default_rng(5)
    dec.set_hf_streams_per_cta(32)
    try:
        for _ in range(12):
            m = bytearray(data)
            for pos in rng.integers(len(m) // 2, len(m), size=3):
                m[pos] ^= 1 << int(rng.integers(0, 8))
            try:
                dec.decode(bytes(m))
            except jxl_oxide_b200.JxlError:
                pass
        dec.decode(bytes(data))  # the decoder keeps working
    finally:
        dec.set_hf_streams_per_cta(0)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_write_to_device_matches_write_to_buffer(dec, dtype):
    """jxlb_frame_write_to_device: the packed frame stays in HBM (input of the NCCL gather, BASELINE config #5)."""
    import jxl_oxide_b200
    import torch
    dec.decode(fixture_bytes("sunset_logo", "input.jxl"))  # orientation 7, alpha
    for orientation in (0, 1, 6):
        host = dec.frame_to_buffer(0, dtype, orientation)
        dev = dec.frame_to_torch(0, dtype, orientation)
        assert dev.is_cuda and tuple(dev.shape) == host.shape
        got = dev.cpu().view(torch.uint8).numpy().view(dtype).reshape(host.shape)
        assert np.array_equal(got.view(np.uint8), host.view(np.uint8))
    # a host pointer is refused with an error value, not dereferenced on the device
    pinned = np.empty(host.shape, dtype=dtype)
    rc = dec._L.jxlb_frame_write_to_device(dec._h, 0, {1: 0, 2: 1, 4: 2}[np.dtype(dtype).itemsize], 0, pinned.ctypes.data, pinned.nbytes)
    assert rc != jxl_oxide_b200.OK


def test_issue_24_one_pixel_vardct_animation(dec, oracle):
    """The reference's 1 x 1 VarDCT animation (its golden buffer pins the oracle in test_oracle_golden.py): every
    keyframe identical to the oracle on the device."""
    data = fixture_bytes("issue_24", "input.jxl")
    dec.decode(data)
    img = oracle.OracleImage(data)
    assert dec.num_frames() == img.num_frames == 9
    for i in range(9):
        got, want = dec.frame_planar(i), img.frame(i)[0]
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("iters", [0, 1, 3])
def test_epf_iteration_counts(dec, oracle, iters):
    """Restoration filter with 0 / 1 / 3 EPF iterations (the all-default filter of the other synthetic frames has 2):
    3 iterations add the 12-neighbour step 0; fused production kernel and the stage-by-stage path against the oracle."""
    data = bench.synth_frame(1000, 600, 7, extra=("--epf-iters", str(iters)))
    img = oracle.OracleImage(data, threads=8)
    want = img.frame(0)[0]
    for fused in (True, False):
        dec.set_fuse_filters(fused)
        try:
            dec.decode(data)
            got = dec.frame_planar(0)
        finally:
            dec.set_fuse_filters(True)
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"fused={fused}"


@pytest.mark.parametrize("streams", [0, 16, 32, 128])
def test_hf_presets_on_the_device(dec, oracle, streams):
    """Several HF presets (synthetic: no reference fixture has more than one). Their cluster maps (5 x 495 x 15 B = 37 KB)
    exceed what the one-warp-per-stream kernel stages, so every value here, 0, 16 and 32 included, runs the
    thread-per-stream kernel, which reads them from global memory."""
    data = bench.synth_frame(1000, 600, 7, extra=("--hf-presets", "5", "--passes", "2"))
    if streams:
        _check(dec, oracle, data, streams)
    else:
        dec.decode(data)
        got, want = dec.frame_planar(0), oracle.OracleImage(data, threads=8).frame(0)[0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_genshin_ycbcr_420_default_schedule(dec, oracle):
    """Full-size 4:2:0 JPEG transcode on the default kernels (the schedule variants are covered by test_hf_lanes_fixture)."""
    data = fixture_bytes("genshin_ycbcr_420", "input.jxl")
    dec.decode(data)
    got, want = dec.frame_planar(0), oracle.OracleImage(data, threads=8).frame(0)[0]
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
