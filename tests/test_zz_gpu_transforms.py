"""GPU parity on frames that hold all 27 VarDCT transform types (tools/synth_enc.cc --all-types) or one type tiled over
the whole frame (--only-type): the only frames that reach the `huge` size class of the inverse transforms
(idct_large_kernel with 256-point lines), HF orders 10-12 (DCT128 .. DCT256) and non-zero contexts of 128 to 1024 blocks.

Every comparison is with the oracle: HF coefficients as integers, every other stage and the final pixels at 0 ULP. The
oracle's own transforms at these sizes are checked against float64 in tests/test_transform_types.py. The file sorts
after the product-default GPU tests, so a blocked kernel here ends the run with every other result already out.
"""
import ctypes

import numpy as np
import pytest

import bench

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

ALL_TYPES_FRAMES = [((1000, 600), 7), ((2600, 700), 5)]
STAGES_F32 = ["lf", "hf_dequant", "idct", "pre_filter", "gaborish", "epf", "rgb"]
# DCT16x8 (the smallest medium shape), DCT64x32 and the six largest types
ONLY_TYPES = [6, 19, 21, 22, 23, 24, 25, 26]


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


def _all_types(size, seed, extra=()):
    return bench.synth_frame(size[0], size[1], seed, extra=("--all-types",) + tuple(extra))


def _same_bits(got, want, what):
    assert got.shape == want.shape, what
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), what


def _check_fused_and_stages(dec, oracle, data):
    """Production path (dequantisation inside the inverse transforms, fused filter chain) on the final pixels, then the
    stage-by-stage path (separate dequantisation kernel, unfused filters) at every stage."""
    img = oracle.OracleImage(data, threads=8, capture=True)
    want = img.frame(0)[0]
    dec.set_capture(False)
    dec.set_fuse_filters(True)
    dec.decode(data)
    _same_bits(dec.frame_planar(0), want, "fused path")
    dec.set_fuse_filters(False)
    dec.set_capture(True)
    try:
        dec.decode(data)
        for g, w in zip(dec.stage("hf_coeff", np.int32), img.stage("hf_coeff", np.int32)):
            assert np.array_equal(g, w), "HF coefficient decode differs"
        for st in STAGES_F32:
            gs, ws = dec.stage(st), img.stage(st)
            assert len(gs) == len(ws) == 3, st
            for c, (g, w) in enumerate(zip(gs, ws)):
                _same_bits(g, w, f"stage {st} channel {c}")
        _same_bits(dec.frame_planar(0), want, "stage-by-stage path")
    finally:
        dec.set_capture(False)
        dec.set_fuse_filters(True)
    img.close()


@pytest.mark.parametrize("size,seed", ALL_TYPES_FRAMES)
def test_all_types_fused_and_stagewise(dec, oracle, size, seed):
    _check_fused_and_stages(dec, oracle, _all_types(size, seed))


@pytest.mark.parametrize("ttype", ONLY_TYPES)
def test_one_type_fills_the_work_lists(dec, oracle, ttype):
    # every group tiled with one type: its size class's work list (items[3] for the huge types) at capacity
    _check_fused_and_stages(dec, oracle, bench.synth_frame(1000, 600, 3, extra=("--only-type", str(ttype))))


@pytest.mark.parametrize("streams", [8, 16, 32, 64, 128])
@pytest.mark.parametrize("extra", [(), ("--passes", "3"), ("--hf-presets", "5")], ids=["one_pass", "passes3", "presets5"])
def test_all_types_hf_schedules(dec, oracle, extra, streams):
    """HF streams per CTA: up to 32 one warp per stream (decode_hf_warp_kernel), 64 and 128 one thread per stream
    (decode_hf_lanes_kernel); five HF presets' cluster maps exceed the warp kernel's staging budget and run the
    thread-per-stream kernel at every setting."""
    data = _all_types((1000, 600), 7, extra)
    img = oracle.OracleImage(data, threads=8, capture=True)
    want, want_coeff = img.frame(0)[0], img.stage("hf_coeff", np.int32)
    img.close()
    dec.set_hf_streams_per_cta(streams)
    dec.set_capture(True)
    try:
        dec.decode(data)
        for g, w in zip(dec.stage("hf_coeff", np.int32), want_coeff):
            assert np.array_equal(g, w), "HF coefficient decode differs"
        _same_bits(dec.frame_planar(0), want, "final pixels")
    finally:
        dec.set_capture(False)
        dec.set_hf_streams_per_cta(0)


@pytest.mark.parametrize("size,seed", ALL_TYPES_FRAMES)
def test_all_types_stage_entry_points(oracle, size, seed):
    """jxlb_decode_hf_groups / jxlb_dequant_idct on caller-owned device planes."""
    import jxl_oxide_b200 as J
    data = _all_types(size, seed)
    img = oracle.OracleImage(data, threads=8, capture=True)
    want_coeff, want_idct = img.stage("hf_coeff", np.int32), img.stage("idct", np.float32)
    img.close()
    d = J.Decoder(0)
    try:
        coeff = d.decode_hf_groups(data)
        assert len(coeff) == 3
        for g, w in zip(coeff, want_coeff):
            assert tuple(g.shape) == w.shape and np.array_equal(g.cpu().numpy(), w)
        out = d.dequant_idct(data)
        assert len(out) == 3
        for g, w in zip(out, want_idct):
            _same_bits(g.cpu().numpy(), w, "dequant_idct")
    finally:
        d.close()


def test_all_types_pipeline_planar_f32(oracle):
    """The frame pipeline with its default HF schedule (thread per stream), several frames in flight."""
    import jxl_oxide_b200 as J
    datas = [_all_types(size, seed) for size, seed in ALL_TYPES_FRAMES] + [_all_types((1000, 600), 7, ("--passes", "3"))]
    want = []
    for d in datas:
        img = oracle.OracleImage(d, threads=16)
        want.append(img.frame(0)[0])
        img.close()
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for rep in range(2):
            for i, d in enumerate(datas):
                p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=10 * rep + i)
        seen = 0
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            w = want[tag % 10]
            assert nbytes == w.nbytes
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=np.float32).reshape(w.shape).copy()
            p.release_output(addr)
            _same_bits(got, w, f"pipeline frame {tag}")
            seen += 1
        assert seen == 2 * len(datas)
    finally:
        p.close()
