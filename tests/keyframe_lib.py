"""ctypes wrapper around the oracle's keyframe decode (tests/emu/keyframes.mk): a keyframe decoded from its own segment
on the CPU, as jxlb_decode_keyframe does on the GPU. Test infrastructure only."""
import ctypes
import os
import subprocess
import sys

import numpy as np

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))
import synth_anim  # noqa: E402

_LIB = None

ANIMATIONS = ["issue_24", "animation_icos4d", "animation_newtons_cradle", "animation_spline"]
# every fixture directory holding one input.jxl that the oracle decodes, animations included
FIXTURES = sorted(d for d in os.listdir(GOLDEN) if os.path.exists(os.path.join(GOLDEN, d, "input.jxl")))
MODES = ["independent", "chain", "mixed"]


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu"), "-f", "keyframes.mk"])
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libjxlkeyframes.so"))
        u32p = ctypes.POINTER(ctypes.c_uint32)
        L.jxlk_segments.argtypes = [ctypes.c_char_p, ctypes.c_size_t, u32p, u32p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        L.jxlk_decode_keyframe.restype = ctypes.c_void_p
        L.jxlk_decode_keyframe.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                           ctypes.c_char_p, ctypes.c_size_t]
        L.jxlk_frame_info.argtypes = [ctypes.c_void_p, u32p, u32p, u32p]
        L.jxlk_frame_channel.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.jxlk_free.argtypes = [ctypes.c_void_p]
        _LIB = L
    return _LIB


def fixture(name):
    with open(os.path.join(GOLDEN, name, "input.jxl"), "rb") as f:
        return f.read()


def animation(mode, frames=7, width=300, height=200, seed=1):
    return synth_anim.synth_animation(width, height, frames, mode, seed)


def segments(data):
    """[(first keyframe, keyframe count)] per segment and the index's error code."""
    first, count = (ctypes.c_uint32 * 4096)(), (ctypes.c_uint32 * 4096)()
    err = ctypes.c_int()
    n = lib().jxlk_segments(data, len(data), first, count, 4096, ctypes.byref(err))
    if n < 0:
        raise oracle_lib.OracleError(err.value, "cannot index the image")
    return [(first[i], count[i]) for i in range(n)], err.value


def decode_keyframe(data, k, threads=4):
    """Keyframe k decoded from its own segment on the oracle: (channels, height, width) float32."""
    L = lib()
    status = ctypes.c_int()
    err = ctypes.create_string_buffer(512)
    h = L.jxlk_decode_keyframe(data, len(data), k, threads, ctypes.byref(status), err, 512)
    if not h:
        raise oracle_lib.OracleError(status.value, err.value.decode())
    try:
        w, hh, n = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        L.jxlk_frame_info(h, ctypes.byref(w), ctypes.byref(hh), ctypes.byref(n))
        out = np.empty((n.value, hh.value, w.value), dtype=np.float32)
        for c in range(n.value):
            L.jxlk_frame_channel(h, c, out[c].ctypes.data)
        return out
    finally:
        L.jxlk_free(h)
