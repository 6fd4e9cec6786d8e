"""GPU tests of the stream entry points that predate the write specs (jxlb_frame_write_to_buffer / _to_device through
Decoder.frame_to_buffer / frame_to_torch, and pipeline out_mode 2, 3 and 4): byte for byte against the numpy model of
tests/write_layouts_lib.py for the stream layout with spot colours mixed, applied to the frame's planes as
jxlb_frame_channel_to_host returns them."""
import ctypes

import numpy as np
import pytest

import write_layouts_lib as W
from test_zz_gpu_write_layouts import ORIENTATIONS, _decoder, _synth

pytestmark = pytest.mark.gpu

# more spot colours than the packer takes in its parameter block, on channels that fit it
NINE_SPOTS = (67, 45, ["alpha:8:0:1"] + ["spot:8:0:1"] * 9)


@pytest.mark.parametrize("name", ["spot", "cmyk_layers", "alpha_triangles", "bench_oriented_brg", "animation_spline", "nine_spots"])
def test_write_to_buffer_matches_the_model(tmp_path, name):
    import torch
    import jxl_oxide_b200 as J
    data = _synth(tmp_path, *NINE_SPOTS) if name == "nine_spots" else W.fixture(name)
    hdr = W.HostImage(data, header_only=True)
    dec = _decoder()
    dec.decode(data)
    planes = dec.frame_planar(0)
    num_color = dec.frame_info(0).num_color
    for dtype in W.DTYPES:
        for o in [0] + list(ORIENTATIONS):
            want = W.model(hdr, 0, W.STREAM, dtype, o, True, planes, num_color)
            got = dec.frame_to_buffer(0, dtype=dtype, orientation=o)
            assert got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8)), (np.dtype(dtype).name, o)
            dev = dec.frame_to_torch(0, dtype=dtype, orientation=o)
            assert np.array_equal(dev.cpu().numpy().view(np.uint8), want.view(np.uint8)), (np.dtype(dtype).name, o)
    p = J.Pipeline(0, workers=2, heavy_frames=2)
    try:
        for mode, dtype in ((J.Pipeline.OUT_U8, np.uint8), (J.Pipeline.OUT_U16, np.uint16)):
            want = W.model(hdr, 0, W.STREAM, dtype, 0, True, planes, num_color)
            host = np.zeros_like(want)
            p.submit(data, out=host, mode=mode)
            p.wait()
            assert np.array_equal(host.view(np.uint8), want.view(np.uint8)), mode
            p.submit(data, mode=mode)  # into the pipeline's ring
            _, addr, nbytes = p.wait(want_output=True)
            assert nbytes == want.nbytes and ctypes.string_at(addr, nbytes) == want.tobytes(), mode
            p.release_output(addr)
        want = W.model(hdr, 0, W.STREAM, np.uint8, 0, True, planes, num_color)
        dev = torch.empty(want.shape, dtype=torch.uint8, device="cuda:0")
        p.submit(data, out=dev, mode=J.Pipeline.OUT_U8_DEVICE)
        p.wait()
        assert np.array_equal(dev.cpu().numpy(), want)
    finally:
        p.close()
