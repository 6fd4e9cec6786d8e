"""CPU tests of the output layouts (jxlb_frame_write_ex): the planner's channel selection against a model of
ImageStream::from_render (fb.rs:184-286), the packer's per-sample code (kernels/pack.cuh, host build) against a numpy
model on oracle planes, and the argument checks of the write plan and the C ABI."""
import ctypes
import subprocess

import numpy as np
import pytest

import bench
import write_layouts_lib as W

# synthetic frames: many extra channels (more than the old packer's 8 planes), spot colours, odd shapes
SYNTH = [
    (257, 129, ["alpha:8:0:1", "spot:10:0:1", "spot:8:0:1"] + ["unknown:8:0:1"] * 9),
    (1, 33, ["alpha:8:0:1", "spot:8:0:1"]),
    (33, 1, ["spot:12:0:1", "alpha:8:0:1"]),
]


def synth(tmp_path, w, h, extras, seed=3):
    out = str(tmp_path / "s.jxl")
    subprocess.check_call([bench.synth_tool(), "--modular", "--width", str(w), "--height", str(h), "--seed", str(seed), "-o", out] +
                          [a for e in extras for a in ("--extra", e)], stderr=subprocess.DEVNULL)
    with open(out, "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def stills():
    return {name: W.HostImage(W.fixture(name)) for name in W.STILLS}


@pytest.mark.parametrize("name", W.STILLS)
def test_channel_selection_follows_the_reference(stills, name):
    img = stills[name]
    for frame in range(img.num_frames):
        num_color = img.frame_info(frame)[3]
        for layout in W.LAYOUTS:
            for spot in (True, False):
                want_ch, want_sp = W.select(num_color, img.extra, img.icc_is_cmyk, img.grayscale, layout, spot)
                rc, ch, sp, _ = img.plan(frame, layout, np.uint8, 0, spot)
                assert rc == 0
                assert (ch, sp) == (want_ch, [c for c, _ in want_sp]), (layout, spot)


def test_fixtures_cover_every_selection_rule(stills):
    """The fixtures hold a CMYK image with a black channel, alpha channels and spot colours, so that each rule is exercised."""
    assert stills["cmyk_layers"].icc_is_cmyk and any(t == W.EC_BLACK for t, _ in stills["cmyk_layers"].extra)
    assert any(t == W.EC_SPOT for t, _ in stills["spot"].extra)
    assert any(t == W.EC_ALPHA for t, _ in stills["alpha_triangles"].extra)
    assert stills["grayscale"].grayscale and stills["bench_oriented_brg"].orientation != 1


def test_stream_layout_is_the_existing_stream(stills):
    """Layout 0 with spot colours on writes what the oracle's ImageStream::write_to_buffer writes, byte for byte."""
    import oracle_lib
    for name in W.STILLS:
        o = oracle_lib.OracleImage(W.fixture(name), threads=4)
        for dtype in W.DTYPES:
            want = o.frame_to_buffer(0, dtype=dtype)
            got = stills[name].pack(0, W.STREAM, dtype, 0, True)
            assert np.array_equal(got.view(np.uint8), want.reshape(-1).view(np.uint8)), (name, dtype)


def _check_all(img, frames, orientations=range(1, 9)):
    for frame in frames:
        planes = img.planes(frame)
        for layout in W.LAYOUTS:
            for spot in (True, False):
                for dtype in W.DTYPES:
                    for o in orientations:
                        want = W.model(img, frame, layout, dtype, o, spot, planes)
                        got = img.pack(frame, layout, dtype, o, spot)
                        assert np.array_equal(got.view(np.uint8), want.reshape(-1).view(np.uint8)), (frame, layout, spot, dtype, o)


@pytest.mark.parametrize("name", W.STILLS)
def test_host_packer_matches_the_model(stills, name):
    _check_all(stills[name], [0])


@pytest.mark.parametrize("w,h,extras", SYNTH)
def test_host_packer_on_odd_shapes_and_many_extra_channels(tmp_path, w, h, extras):
    img = W.HostImage(synth(tmp_path, w, h, extras))
    assert len(img.extra) == len(extras)
    _check_all(img, [0])


def test_write_plan_rejects_bad_specs(stills):
    img = stills["alpha_triangles"]
    assert img.plan(0, 0)[0] == 0
    for layout in (-1, 4):
        assert img.plan(0, layout)[0] == 5  # kErrInvalidArg
    for st in (-1, 3):
        assert img.plan(0, W.STREAM, st)[0] == 5
    for o in (-1, 9):
        assert img.plan(0, W.STREAM, np.uint8, o)[0] == 5
    w, h, _, _ = img.frame_info(0)
    rc, ch, _, nbytes = img.plan(0, W.ALL_PLANAR, np.uint16, 6)
    assert rc == 0 and nbytes == w * h * len(ch) * 2


def test_abi_rejects_bad_arguments_without_a_device():
    import jxl_oxide_b200 as J
    L = J.load_library()
    spec = J.write_spec("stream", np.uint8)
    n, nbytes = ctypes.c_uint32(), ctypes.c_uint64()
    buf = ctypes.create_string_buffer(16)
    assert L.jxlb_frame_write_size(None, 0, ctypes.byref(spec), ctypes.byref(n), ctypes.byref(nbytes)) == J.ERR_INVALID_ARG
    assert L.jxlb_frame_write_ex(None, 0, ctypes.byref(spec), buf, 16, 0) == J.ERR_INVALID_ARG
    assert L.jxlb_pipeline_submit_ex(None, None, 0, 0, ctypes.byref(spec), None, 0, 0, 0) == J.ERR_INVALID_ARG
    assert L.jxlb_pipeline_submit_keyframes_ex(None, None, 0, 0, ctypes.byref(spec), None, 0, 0, 0) == J.ERR_INVALID_ARG
    assert J.write_spec("all_channels", np.float32, 6, False).layout == J.LAYOUT_ALL_INTERLEAVED
