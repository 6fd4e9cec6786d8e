"""Models of the reference's output layouts (crates/jxl-oxide/src/fb.rs, lib.rs:1133-1198) in numpy, and a ctypes
wrapper of tests/emu/pack.mk (the oracle with the packer's host build). Test infrastructure only."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

STREAM, STREAM_NO_ALPHA, ALL_INTERLEAVED, ALL_PLANAR = range(4)
LAYOUTS = [STREAM, STREAM_NO_ALPHA, ALL_INTERLEAVED, ALL_PLANAR]
DTYPES = [np.uint8, np.uint16, np.float32]
SAMPLE_TYPE = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2}
# extra channel types (jxl-image/src/lib.rs:303-345)
EC_ALPHA, EC_SPOT, EC_BLACK = 0, 2, 4

STILLS = ["spot", "cmyk_layers", "alpha_nonpremultiplied", "alpha_premultiplied", "alpha_triangles", "grayalpha", "blendmodes",
          "grayscale", "bench_oriented_brg"]
ANIMATIONS = ["animation_icos4d", "animation_newtons_cradle", "animation_spline", "issue_24"]


def fixture(name):
    with open(os.path.join(GOLDEN, name, "input.jxl"), "rb") as f:
        return f.read()


def select(num_color, extra, icc_is_cmyk, grayscale, layout, spot_colours):
    """ImageStream::from_render (fb.rs:184-286) / image_all_channels: the channels written, in order, and the spot
    colour channels mixed in. `extra`: [(type, (r, g, b, solidity))] in header order."""
    if layout in (ALL_INTERLEAVED, ALL_PLANAR):
        return list(range(num_color + len(extra))), []
    channels = list(range(num_color))
    if icc_is_cmyk:
        channels += [num_color + e for e, (t, _) in enumerate(extra) if t == EC_BLACK][:1]
    if layout == STREAM:
        channels += [num_color + e for e, (t, _) in enumerate(extra) if t == EC_ALPHA][:1]
    spots = []
    if spot_colours and num_color == 3 and not grayscale:
        spots = [(num_color + e, s) for e, (t, s) in enumerate(extra) if t == EC_SPOT]
    return channels, spots


def source_coords(orientation, ow, oh):
    """(sy, sx) index arrays of the stored sample each output sample reads (to_original_coord, fb.rs:383-397)."""
    y, x = np.mgrid[0:oh, 0:ow]
    sx, sy = {1: (x, y), 2: (ow - x - 1, y), 3: (ow - x - 1, oh - y - 1), 4: (x, oh - y - 1), 5: (y, x), 6: (y, ow - x - 1),
              7: (oh - y - 1, ow - x - 1), 8: (oh - y - 1, x)}[orientation]
    return sy, sx


def pack(planes, channels, spots, orientation, dtype, planar):
    """The written samples: spot colours mixed into channels 0..2 in f32 (fb.rs:335-362), orientation applied, then the
    sample conversion of fb.rs:436-520. (h, w, c) interleaved or (c, h, w) planar."""
    one = np.float32(1.0)
    out = []
    for i, c in enumerate(channels):
        v = planes[c].astype(np.float32)
        if i < 3:
            for sc, (r, g, b, solidity) in spots:
                mix = planes[sc] * np.float32(solidity)
                v = np.float32((r, g, b)[i]) * mix + v * (one - mix)
        out.append(v)
    h, w = planes[0].shape
    ow, oh = (h, w) if orientation >= 5 else (w, h)
    sy, sx = source_coords(orientation, ow, oh)
    arr = np.stack(out)[:, sy, sx]
    if np.dtype(dtype) != np.float32:
        hi = np.float32(255.0 if np.dtype(dtype) == np.uint8 else 65535.0)
        t = arr * hi + np.float32(0.5)
        t = np.where(t < 0, np.float32(0), np.where(t > hi, hi, t))  # NaN stays NaN, then becomes 0
        arr = np.where(np.isnan(t), np.float32(0), t).astype(np.uint32).astype(dtype)
    return np.ascontiguousarray(arr if planar else arr.transpose(1, 2, 0))


_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu"), "-f", "pack.mk"])
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libjxlpack.so"))
        vp, u32p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32)
        L.jxlw_decode.restype = vp
        L.jxlw_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_char_p,
                                  ctypes.c_size_t]
        L.jxlw_read_header.restype = vp
        L.jxlw_read_header.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
        L.jxlw_header.argtypes = [vp, u32p, u32p, u32p, u32p]
        L.jxlw_extra_channel.argtypes = [vp, ctypes.c_int, u32p, ctypes.POINTER(ctypes.c_float)]
        L.jxlw_num_frames.argtypes = [vp]
        L.jxlw_frame_info.argtypes = [vp, ctypes.c_int, u32p, u32p, u32p, u32p]
        L.jxlw_frame_channel.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp]
        L.jxlw_plan.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, u32p, u32p, u32p, u32p,
                                ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint64), ctypes.c_char_p, ctypes.c_size_t]
        L.jxlw_pack.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
        L.jxlw_free.argtypes = [vp]
        _LIB = L
    return _LIB


class HostImage:
    """An image decoded by the oracle, with the planner's write plan and the packer's host build. header_only: the image
    header alone, for the channel selection of frames decoded on the device."""

    def __init__(self, data, threads=4, header_only=False):
        L = lib()
        status = ctypes.c_int()
        err = ctypes.create_string_buffer(512)
        if header_only:
            self._h = L.jxlw_read_header(data, len(data))
        else:
            self._h = L.jxlw_decode(data, len(data), threads, ctypes.byref(status), err, 512)
        if not self._h:
            raise RuntimeError(f"[{status.value}] {err.value.decode()}")
        cmyk, gray, orient, n = (ctypes.c_uint32() for _ in range(4))
        L.jxlw_header(self._h, ctypes.byref(cmyk), ctypes.byref(gray), ctypes.byref(orient), ctypes.byref(n))
        self.icc_is_cmyk, self.grayscale, self.orientation = bool(cmyk.value), bool(gray.value), orient.value
        self.extra = []
        for e in range(n.value):
            t, spot = ctypes.c_uint32(), (ctypes.c_float * 4)()
            L.jxlw_extra_channel(self._h, e, ctypes.byref(t), spot)
            self.extra.append((t.value, tuple(spot)))
        self.num_frames = L.jxlw_num_frames(self._h)

    def frame_info(self, frame):
        w, h, n, nc = (ctypes.c_uint32() for _ in range(4))
        lib().jxlw_frame_info(self._h, frame, ctypes.byref(w), ctypes.byref(h), ctypes.byref(n), ctypes.byref(nc))
        return w.value, h.value, n.value, nc.value

    def planes(self, frame):
        w, h, n, _ = self.frame_info(frame)
        out = np.empty((n, h, w), dtype=np.float32)
        for c in range(n):
            lib().jxlw_frame_channel(self._h, frame, c, out[c].ctypes.data)
        return out

    def plan(self, frame, layout, dtype=np.uint8, orientation=0, spot_colours=True):
        """(status, channels, spot channels, bytes) of plan_write."""
        cap = 512
        ch, sp = (ctypes.c_uint32 * cap)(), (ctypes.c_uint32 * cap)()
        nch, nsp, nbytes = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint64()
        err = ctypes.create_string_buffer(256)
        st = SAMPLE_TYPE.get(np.dtype(dtype), 9) if not isinstance(dtype, int) else dtype
        rc = lib().jxlw_plan(self._h, frame, layout, st, orientation, int(spot_colours), ch, ctypes.byref(nch), sp, ctypes.byref(nsp),
                             cap, ctypes.byref(nbytes), err, 256)
        return rc, list(ch[:nch.value]), list(sp[:nsp.value]), nbytes.value

    def pack(self, frame, layout, dtype, orientation, spot_colours):
        rc, _, _, nbytes = self.plan(frame, layout, dtype, orientation, spot_colours)
        assert rc == 0
        out = np.empty(nbytes // np.dtype(dtype).itemsize, dtype=dtype)
        assert lib().jxlw_pack(self._h, frame, layout, SAMPLE_TYPE[np.dtype(dtype)], orientation, int(spot_colours), out.ctypes.data) == 0
        return out

    def close(self):
        if self._h:
            lib().jxlw_free(self._h)
            self._h = None

    def __del__(self):
        self.close()


def model(img, frame, layout, dtype, orientation, spot_colours, planes=None, num_color=None):
    """The numpy model's output for frame `frame` of a HostImage (or, given `planes` and `num_color`, of a frame decoded
    elsewhere and the HostImage of its header)."""
    if planes is None:
        planes = img.planes(frame)
    if num_color is None:
        num_color = img.frame_info(frame)[3]
    channels, spots = select(num_color, img.extra, img.icc_is_cmyk, img.grayscale, layout, spot_colours)
    return pack(planes, channels, spots, orientation or img.orientation, dtype, layout == ALL_PLANAR)
