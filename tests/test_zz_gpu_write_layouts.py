"""GPU tests of the output layouts (kernels/pack.cu through jxlb_frame_write_ex, the pipeline's spec submissions and the
Render methods): every layout x orientation 1..8 x u8 / u16 / f32, spot colours on and off, byte for byte against the
numpy model of tests/write_layouts_lib.py applied to the frame's planes as jxlb_frame_channel_to_host returns them."""
import ctypes
import subprocess

import numpy as np
import pytest

import bench
import write_layouts_lib as W

pytestmark = pytest.mark.gpu

ORIENTATIONS = range(1, 9)
# odd shapes, and more extra channels than the interleaving kernel of jxlb_frame_write_to_buffer takes
SYNTH = [
    (257, 129, ["alpha:8:0:1", "spot:10:0:1", "spot:8:0:1"] + ["unknown:8:0:1"] * 9),
    (1, 77, ["alpha:8:0:1", "spot:8:0:1"]),
    (77, 1, ["spot:12:0:1", "alpha:8:0:1"]),
    (1, 1, ["alpha:8:0:1"]),
]


def _decoder():
    import jxl_oxide_b200 as J
    return J.Decoder(0)


def _synth(tmp_path, w, h, extras, seed=5):
    out = str(tmp_path / "s.jxl")
    subprocess.check_call([bench.synth_tool(), "--modular", "--width", str(w), "--height", str(h), "--seed", str(seed), "-o", out] +
                          [a for e in extras for a in ("--extra", e)], stderr=subprocess.DEVNULL)
    with open(out, "rb") as f:
        return f.read()


def _check_frame(dec, hdr, frame):
    planes = dec.frame_planar(frame)
    num_color = dec.frame_info(frame).num_color
    for layout in W.LAYOUTS:
        for spot in (True, False):
            for dtype in W.DTYPES:
                for o in ORIENTATIONS:
                    want = W.model(hdr, frame, layout, dtype, o, spot, planes, num_color)
                    got = dec.frame_write(frame, layout, dtype, o, spot)
                    assert got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8)), \
                        (frame, layout, spot, np.dtype(dtype).name, o)


def _frames(n):
    return sorted({0, n // 2, n - 1})


@pytest.mark.parametrize("name", W.STILLS + W.ANIMATIONS)
def test_every_layout_matches_the_model(name):
    data = W.fixture(name)
    hdr = W.HostImage(data, header_only=True)
    dec = _decoder()
    dec.decode(data)
    for frame in _frames(dec.num_frames()):
        _check_frame(dec, hdr, frame)


@pytest.mark.parametrize("w,h,extras", SYNTH)
def test_odd_shapes_and_many_extra_channels(tmp_path, w, h, extras):
    data = _synth(tmp_path, w, h, extras)
    hdr = W.HostImage(data, header_only=True)
    assert len(hdr.extra) == len(extras)
    dec = _decoder()
    dec.decode(data)
    _check_frame(dec, hdr, 0)


@pytest.mark.parametrize("name", ["spot", "cmyk_layers", "alpha_triangles", "bench_oriented_brg", "animation_spline"])
def test_stream_layout_equals_write_to_buffer(name):
    dec = _decoder()
    dec.decode(W.fixture(name))
    for dtype in W.DTYPES:
        for o in [0] + list(ORIENTATIONS):
            want = dec.frame_to_buffer(0, dtype=dtype, orientation=o)
            got = dec.frame_write(0, W.STREAM, dtype, o)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (np.dtype(dtype).name, o)


@pytest.mark.parametrize("name", ["spot", "cmyk_layers", "grayalpha", "bench_oriented_brg"])
def test_device_destination_equals_host(name):
    import torch
    tdt = {np.uint8: torch.uint8, np.uint16: torch.uint16, np.float32: torch.float32}
    dec = _decoder()
    dec.decode(W.fixture(name))
    for layout in W.LAYOUTS:
        for dtype in W.DTYPES:
            for o in (1, 3, 6, 8):
                host = dec.frame_write(0, layout, dtype, o)
                dev = torch.empty(host.shape, dtype=tdt[dtype], device="cuda:0")
                assert dec.frame_write(0, layout, dtype, o, out=dev) is dev
                assert np.array_equal(dev.cpu().numpy().view(np.uint8), host.view(np.uint8)), (layout, np.dtype(dtype).name, o)


def test_bad_arguments_are_rejected():
    import jxl_oxide_b200 as J
    dec = _decoder()
    dec.decode(W.fixture("alpha_triangles"))
    L, h = dec._L, dec._h
    n, nbytes = ctypes.c_uint32(), ctypes.c_uint64()
    for spec in (J.WriteSpec(4, 0, 0, 1), J.WriteSpec(-1, 0, 0, 1), J.WriteSpec(0, 3, 0, 1), J.WriteSpec(0, 0, 9, 1),
                 J.WriteSpec(0, 0, -1, 1)):
        assert L.jxlb_frame_write_size(h, 0, ctypes.byref(spec), ctypes.byref(n), ctypes.byref(nbytes)) == J.ERR_INVALID_ARG
        buf = np.empty(1 << 20, np.uint8)
        assert L.jxlb_frame_write_ex(h, 0, ctypes.byref(spec), buf.ctypes.data, buf.nbytes, 0) == J.ERR_INVALID_ARG
    spec = J.write_spec("all_channels", np.uint16, 6)
    assert L.jxlb_frame_write_size(h, 0, ctypes.byref(spec), ctypes.byref(n), ctypes.byref(nbytes)) == J.OK
    info = dec.frame_info(0)
    assert n.value == info.num_channels and nbytes.value == info.width * info.height * n.value * 2
    small = np.empty(nbytes.value - 1, np.uint8)
    assert L.jxlb_frame_write_ex(h, 0, ctypes.byref(spec), small.ctypes.data, small.nbytes, 0) == J.ERR_INVALID_ARG
    assert L.jxlb_frame_write_ex(h, 1, ctypes.byref(spec), small.ctypes.data, small.nbytes, 0) == J.ERR_INVALID_ARG
    # host memory passed as a device destination
    big = np.empty(nbytes.value, np.uint8)
    assert L.jxlb_frame_write_ex(h, 0, ctypes.byref(spec), big.ctypes.data, big.nbytes, 1) == J.ERR_INVALID_ARG
    with pytest.raises(ValueError):
        dec.frame_write(0, "stream", np.uint8, out=np.empty((1, 1, 1), np.uint8))


def test_render_methods():
    import jxl_oxide_b200 as J
    data = W.fixture("spot")
    img = J.JxlImage.read(data)
    hdr = W.HostImage(data, header_only=True)
    r = img.render_frame(0)
    planes = r.image_planar()
    nc = r.num_color
    assert np.array_equal(planes, img.decoder.frame_planar(0))  # unchanged: the stored planes
    o = hdr.orientation
    assert np.array_equal(r.image_planar(oriented=True), W.model(hdr, 0, W.ALL_PLANAR, np.float32, o, True, planes, nc))
    assert np.array_equal(r.image_all_channels(), W.model(hdr, 0, W.ALL_INTERLEAVED, np.float32, o, True, planes, nc))
    assert np.array_equal(r.stream(dtype=np.uint8), W.model(hdr, 0, W.STREAM, np.uint8, o, True, planes, nc))
    assert np.array_equal(r.stream(no_alpha=True), W.model(hdr, 0, W.STREAM_NO_ALPHA, np.float32, o, True, planes, nc))
    assert img.set_render_spot_color(False) is img and not img.render_spot_color()
    r = img.render_frame(0)
    assert np.array_equal(r.stream(), W.model(hdr, 0, W.STREAM, np.float32, o, False, planes, nc))
    gray = J.JxlImage.read(W.fixture("grayscale"))
    gray.set_render_spot_color(False)
    gray.set_render_spot_color(True)  # ignored on a grayscale image, as the reference does
    assert not gray.render_spot_color()


SPECS = [("stream", np.uint8, 0, True), ("stream_no_alpha", np.uint16, 6, True), ("all_channels", np.float32, 3, True),
         ("planar", np.float32, 8, False), ("stream", np.float32, 5, False)]


@pytest.mark.parametrize("name", ["spot", "alpha_triangles", "cmyk_layers"])
def test_pipeline_submit_with_a_spec(name):
    import torch
    import jxl_oxide_b200 as J
    data = W.fixture(name)
    dec = _decoder()
    dec.decode(data)
    p = J.Pipeline(0, workers=2, heavy_frames=2)
    try:
        for layout, dtype, o, spot in SPECS:
            want = dec.frame_write(0, layout, dtype, o, spot)
            spec = J.write_spec(layout, dtype, o, spot)
            # device destination
            tdt = {np.uint8: torch.uint8, np.uint16: torch.uint16, np.float32: torch.float32}[dtype]
            dev = torch.empty(want.shape, dtype=tdt, device="cuda:0")
            p.submit(data, out=dev, spec=spec)
            p.wait()
            assert np.array_equal(dev.cpu().numpy().view(np.uint8), want.view(np.uint8)), (layout, o)
            # host destination
            host = np.zeros_like(want)
            p.submit(data, out=host, spec=spec)
            p.wait()
            assert np.array_equal(host.view(np.uint8), want.view(np.uint8)), (layout, o)
            # the ring
            p.submit(data, spec=spec)
            _, addr, nbytes = p.wait(want_output=True)
            assert nbytes == want.nbytes
            assert ctypes.string_at(addr, nbytes) == want.tobytes(), (layout, o)
            p.release_output(addr)
    finally:
        p.close()


@pytest.mark.parametrize("name", ["animation_spline", "issue_24"])
def test_pipeline_keyframes_with_a_spec(name):
    import torch
    import jxl_oxide_b200 as J
    data = W.fixture(name)
    dec = _decoder()
    dec.decode(data)
    nk = dec.num_frames()
    p = J.Pipeline(0, workers=2, heavy_frames=2)
    try:
        for layout, dtype, o, spot in SPECS:
            want = np.stack([dec.frame_write(k, layout, dtype, o, spot) for k in range(nk)])
            spec = J.write_spec(layout, dtype, o, spot)
            tdt = {np.uint8: torch.uint8, np.uint16: torch.uint16, np.float32: torch.float32}[dtype]
            dev = torch.empty(want.shape, dtype=tdt, device="cuda:0")
            p.submit_keyframes(data, out=dev, spec=spec)
            for _ in range(nk):
                p.wait_keyframe()
            assert np.array_equal(dev.cpu().numpy().view(np.uint8), want.view(np.uint8)), (layout, o)
            p.submit_keyframes(data, spec=spec)
            seen = set()
            for _ in range(nk):
                _, k, addr, nbytes = p.wait_keyframe(want_output=True)
                assert nbytes == want[k].nbytes
                assert ctypes.string_at(addr, nbytes) == want[k].tobytes(), (layout, o, k)
                p.release_output(addr)
                seen.add(k)
            assert seen == set(range(nk))
    finally:
        p.close()
