"""CPU tests: the keyframe entry points are exported, mirrored in Python and reject bad arguments without a device."""
import ctypes

import jxl_oxide_b200 as J
import keyframe_lib as K

NAMES = ["jxlb_image_keyframes", "jxlb_decode_keyframe", "jxlb_pipeline_submit_keyframes", "jxlb_pipeline_wait_keyframe"]


def test_keyframe_symbols_are_exported_and_listed():
    L = J.load_library()
    for name in NAMES:
        assert hasattr(L, name)
        assert name in J.EXPORTED_SYMBOLS
    for attr in ("decode_keyframe",):
        assert hasattr(J.Decoder, attr)
    for attr in ("submit_keyframes", "wait_keyframe"):
        assert hasattr(J.Pipeline, attr)
    assert callable(J.image_keyframes)


def test_keyframe_entry_points_reject_bad_arguments():
    L = J.load_library()
    nk, ns = ctypes.c_int32(7), ctypes.c_int32(7)
    assert L.jxlb_image_keyframes(None, 0, ctypes.byref(nk), ctypes.byref(ns)) == J.ERR_INVALID_ARG
    assert (nk.value, ns.value) == (0, 0)
    data = K.fixture("animation_icos4d")
    assert L.jxlb_image_keyframes(data, len(data), None, None) == J.OK  # counts are optional
    assert L.jxlb_decode_keyframe(None, data, len(data), None, 0) == J.ERR_INVALID_ARG
    assert L.jxlb_pipeline_submit_keyframes(None, None, 0, 0, 0, None, 0, 0) == J.ERR_INVALID_ARG
    tag, kf, st = ctypes.c_uint64(), ctypes.c_int32(), ctypes.c_int32()
    assert L.jxlb_pipeline_wait_keyframe(None, ctypes.byref(tag), ctypes.byref(kf), ctypes.byref(st), None, None, None, 0) == J.ERR_INVALID_ARG


def test_image_keyframes_of_a_container_and_a_truncated_header():
    data = K.fixture("issue_24")
    nk, ns, st = J.image_keyframes(data)
    assert nk == 9 and st == J.OK
    L = J.load_library()
    n = ctypes.c_int32(-1)
    assert L.jxlb_image_keyframes(data, 5, ctypes.byref(n), None) != J.OK and n.value == 0
