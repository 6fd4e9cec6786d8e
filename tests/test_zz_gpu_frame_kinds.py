"""GPU tests of the frame kinds of tests/frame_kinds_lib.py: jxlb_decode in every output_colour, jxlb_decode_keyframe for
every keyframe and jxlb_pipeline_submit_keyframes, each against the oracle bit for bit."""
import ctypes

import numpy as np
import pytest

import frame_kinds_lib as F
import jxl_oxide_b200 as J
import oracle_lib

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

NAMES = sorted(F.STREAMS)


def _oracle(data, output_colour=0):
    o = oracle_lib.OracleImage(data, output_colour=output_colour, threads=16)
    return o, [o.frame(k)[0] for k in range(o.num_frames)]


@pytest.mark.parametrize("output_colour", [0, 1, 2])
@pytest.mark.parametrize("name", NAMES)
def test_decode_and_decode_keyframe_match_oracle(name, output_colour):
    data = F.STREAMS[name]
    _, wants = _oracle(data, output_colour)
    full, one = J.Decoder(0), J.Decoder(0)
    full.decode(data, output_colour=output_colour)
    assert full.num_frames() == len(wants)
    for k, want in enumerate(wants):
        got = full.frame_planar(k)
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{name}: keyframe {k} differs"
        one.decode_keyframe(data, k, output_colour=output_colour)
        assert np.array_equal(one.frame_planar(0).view(np.uint32), want.view(np.uint32)), f"{name}: keyframe {k} alone"
    full.close()
    one.close()


def test_pipeline_keyframes_match_oracle():
    pipe = J.Pipeline(0, workers=3, heavy_frames=2)
    jobs = {}
    for name in NAMES:
        o, wants = _oracle(F.STREAMS[name])
        bufs = [o.frame_to_buffer(k, np.uint8) for k in range(o.num_frames)]
        jobs[pipe.submit_keyframes(F.STREAMS[name], mode=2)] = (name, bufs, [])
    while pipe.in_flight:
        tag, k, addr, nbytes = pipe.wait_keyframe(want_output=True)
        name, bufs, seen = jobs[tag]
        got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=np.uint8).reshape(bufs[k].shape).copy()
        pipe.release_output(addr)
        assert np.array_equal(got, bufs[k]), f"{name}: keyframe {k} differs"
        seen.append(k)
    for name, bufs, seen in jobs.values():
        assert sorted(seen) == list(range(len(bufs))), name
    pipe.close()


@pytest.mark.parametrize("name", ["preview_small", "preview_default_header"])
def test_pipeline_submit_still_with_preview(name):
    _, wants = _oracle(F.STREAMS[name])
    out = np.zeros_like(wants[0])
    pipe = J.Pipeline(0, workers=2, heavy_frames=2)
    pipe.submit(F.STREAMS[name], out=out)
    while pipe.in_flight:
        pipe.wait()
    assert np.array_equal(out.view(np.uint32), wants[0].view(np.uint32))
    pipe.close()


def test_icc_blend_onto_a_slot_before_the_transform():
    # refused where the oracle refuses (the frame would be converted before being composed onto an XYB slot); with XYB
    # output the keyframe matches the oracle
    data = F.icc_image([dict(reference=True, save_as=1), dict(crop=F.ICC_SUB, source=1)])
    d = J.Decoder(0)
    for output_colour in (0, 1):
        with pytest.raises(J.JxlError) as e:
            d.decode(data, output_colour=output_colour)
        assert e.value.code == J.ERR_UNSUPPORTED
    d.decode(data, output_colour=2)
    want = _oracle(data, 2)[1][0]
    assert np.array_equal(d.frame_planar(0).view(np.uint32), want.view(np.uint32))
    d.close()
