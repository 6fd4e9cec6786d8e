"""Splines and noise on upsampled VarDCT frames on the device, bit for bit like the oracle: every stage and the final
planes through jxlb_decode, jxlb_decode_keyframe, the frame pipeline (planar f32 and u8), and an 8K frame."""
import ctypes

import numpy as np
import pytest

from test_upsampled_features import bits, encode, up_args

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200, method="thread")]

KINDS = [(w, h, k, f) for (w, h) in [(7, 5), (130, 70), (257, 256), (1000, 600)] for k in (2, 4, 8)
         for f in (("--noise",), ("--splines", "1" if w * h < 100 else "6", "--noise"))]
KINDS += [(1, 1, 2, ()), (1000, 600, 2, ("--noise-zero",)), (1000, 600, 4, ("--splines", "6"))]
IDS = [f"{w}x{h} k{k} " + " ".join(f) for w, h, k, f in KINDS]
STAGES = ["splines", "noise", "upsampled", "rgb"]


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


@pytest.mark.parametrize("w,h,k,feat", KINDS, ids=IDS)
def test_decode_matches_oracle(dec, oracle, tmp_path, w, h, k, feat):
    data = encode(tmp_path, w, h, up_args(k, *feat))
    img = oracle.OracleImage(data, threads=8, capture=True)
    want = img.frame(0)[0]
    dec.set_capture(True)
    try:
        dec.decode(data)
        got = dec.frame_planar(0)
        assert got.shape == want.shape
        assert np.array_equal(bits(got), bits(want))
        for st in STAGES:
            gs, ws = dec.stage(st), img.stage(st)
            assert len(gs) == len(ws), st
            for g, wv in zip(gs, ws):
                assert np.array_equal(bits(g), bits(wv)), st
        assert np.array_equal(dec.frame_to_buffer(0, np.uint8), img.frame_to_buffer(0, np.uint8))
    finally:
        dec.set_capture(False)
    dec.decode(data)  # production path
    assert np.array_equal(bits(dec.frame_planar(0)), bits(want))
    one = __import__("jxl_oxide_b200").Decoder(0)
    try:
        one.decode_keyframe(data, 0)
        assert np.array_equal(bits(one.frame_planar(0)), bits(want))
    finally:
        one.close()


def test_noise_on_a_frame_narrower_than_two_samples_is_refused(dec, tmp_path):
    import jxl_oxide_b200 as J
    with pytest.raises(J.JxlError) as e:
        dec.decode(encode(tmp_path, 1, 1, up_args(2, "--noise")))
    assert e.value.code == J.ERR_UNSUPPORTED
    with pytest.raises(J.JxlError) as e:
        dec.decode(encode(tmp_path, 130, 70, up_args(2, "--dangling-patch", "--noise")))
    assert e.value.code == J.ERR_UNSUPPORTED


def _pipeline_check(J, datas, planar, packed, workers, heavy):
    p = J.Pipeline(0, workers=workers, heavy_frames=heavy)
    try:
        for i, d in enumerate(datas):
            p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=i)
            if packed is not None:
                p.submit(data=d, mode=p.OUT_U8, tag=100 + i)
        seen = 0
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            kind, i = divmod(tag, 100)
            want = planar[i] if kind == 0 else packed[i]
            assert nbytes == want.nbytes, tag
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=want.dtype).reshape(want.shape).copy()
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), tag
            seen += 1
        assert seen == len(datas) * (1 if packed is None else 2)
    finally:
        p.close()


def test_pipeline_outputs_match_oracle(oracle, tmp_path):
    import jxl_oxide_b200 as J
    cases = [c for c in KINDS if c[0] * c[1] > 100]
    datas, planar, packed = [], [], []
    for i, (w, h, k, feat) in enumerate(cases):
        d = encode(tmp_path, w, h, up_args(k, *feat), seed=i + 3)
        img = oracle.OracleImage(d, threads=8)
        datas.append(d)
        planar.append(img.frame(0)[0])
        packed.append(img.frame_to_buffer(0, np.uint8))
        img.close()
    _pipeline_check(J, datas, planar, packed, 4, 2)


def test_8k_frame_with_upsampling_2(dec, oracle, tmp_path):
    """7680x4320 coded at 3840x2160, with splines past the coded edge and noise from the 8K field, through jxlb_decode
    and a pipeline at the bench's 64 workers and 16 heavy slots."""
    import jxl_oxide_b200 as J
    data = encode(tmp_path, 7680, 4320, up_args(2, "--splines", "12", "--noise"))
    want = oracle.OracleImage(data, threads=16).frame(0)[0]
    dec.decode(data)
    assert np.array_equal(bits(dec.frame_planar(0)), bits(want))
    _pipeline_check(J, [data] * 3, [want] * 3, None, 64, 16)
