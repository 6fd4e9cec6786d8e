"""ctypes wrapper around the CPU oracle (oracle/_build/libjxloracle.so). Test infrastructure only."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])


def lib():
    global _LIB
    if _LIB is None:
        L = _load(os.path.join(ROOT, "oracle", "_build", "libjxloracle.so"), os.path.join(ROOT, "oracle"))
        _LIB = L
    return _LIB


_EMU_LIB = None


def emu_lib():
    """The oracle rebuilt around tests/emu/emu_backend.cc (always rebuilt through make: it tracks the kernel headers)."""
    global _EMU_LIB
    if _EMU_LIB is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")])
        _EMU_LIB = _load(os.path.join(ROOT, "tests", "emu", "_build", "libjxlemu.so"), None)
    return _EMU_LIB


def _load(path, make_dir):
    if not os.path.exists(path):
        subprocess.check_call(["make", "-s", "-C", make_dir])
    L = ctypes.CDLL(path)
    L.jxlo_decode.restype = ctypes.c_void_p
    L.jxlo_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                              ctypes.POINTER(ctypes.c_int), ctypes.c_char_p, ctypes.c_size_t]
    L.jxlo_num_frames.argtypes = [ctypes.c_void_p]
    L.jxlo_image_info.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint32)] * 6
    L.jxlo_image_orientation.argtypes = [ctypes.c_void_p]
    L.jxlo_image_orientation.restype = ctypes.c_uint32
    L.jxlo_frame_info.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.POINTER(ctypes.c_uint32)] * 5
    L.jxlo_frame_channel.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.jxlo_frame_write_to_buffer.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.jxlo_frame_write_to_buffer.restype = ctypes.c_size_t
    L.jxlo_image_original_icc.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    L.jxlo_image_original_icc.restype = ctypes.c_size_t
    L.jxlo_icc_to_enum.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32)]
    L.jxlo_frame_stream_channels.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.jxlo_frame_stream_channels.restype = ctypes.c_uint32
    L.jxlo_stage.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint32),
                             ctypes.POINTER(ctypes.c_uint32), ctypes.c_void_p]
    L.jxlo_frame_filters.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]
    L.jxlo_free.argtypes = [ctypes.c_void_p]
    return L


def icc_to_enum(icc: bytes):
    """(status, dict) of the ICC recognition rules: status 0 = an enum encoding describes the profile."""
    out = (ctypes.c_uint32 * 7)()
    st = lib().jxlo_icc_to_enum(icc, len(icc), out)
    keys = ("colour_space", "white_point", "primaries", "tf", "gamma", "gamma_inverted", "rendering_intent")
    return st, dict(zip(keys, [int(x) for x in out]))


class OracleError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"oracle decode failed ({code}): {msg}")
        self.code = code


class OracleImage:
    def __init__(self, data: bytes, output_colour=0, threads=1, capture=False, emu=False):
        L = self._L = emu_lib() if emu else lib()
        status = ctypes.c_int(0)
        err = ctypes.create_string_buffer(512)
        self._h = L.jxlo_decode(data, len(data), output_colour, threads, int(capture), ctypes.byref(status), err, 512)
        if not self._h:
            raise OracleError(status.value, err.value.decode())
        v = [ctypes.c_uint32() for _ in range(6)]
        L.jxlo_image_info(self._h, *[ctypes.byref(x) for x in v])
        self.width, self.height, self.bits, self.num_extra, self.xyb, self.gray = [x.value for x in v]
        self.num_frames = L.jxlo_num_frames(self._h)
        self.orientation = L.jxlo_image_orientation(self._h)

    def frame(self, idx=0):
        L = self._L
        v = [ctypes.c_uint32() for _ in range(5)]
        L.jxlo_frame_info(self._h, idx, *[ctypes.byref(x) for x in v])
        w, h, nch, ncol, vardct = [x.value for x in v]
        out = np.empty((nch, h, w), dtype=np.float32)
        for c in range(nch):
            L.jxlo_frame_channel(self._h, idx, c, out[c].ctypes.data)
        return out, ncol, bool(vardct)

    def frame_filters(self, idx=0):
        """(Gaborish on, EPF iteration count) of the frame's header."""
        gab, iters = ctypes.c_uint32(), ctypes.c_uint32()
        self._L.jxlo_frame_filters(self._h, idx, ctypes.byref(gab), ctypes.byref(iters))
        return bool(gab.value), int(iters.value)

    def original_icc(self):
        L = self._L
        n = L.jxlo_image_original_icc(self._h, None, 0)
        buf = ctypes.create_string_buffer(max(n, 1))
        L.jxlo_image_original_icc(self._h, buf, n)
        return buf.raw[:n]

    def frame_to_buffer(self, idx=0, dtype=np.uint8, orientation=0):
        """ImageStream::write_to_buffer: (height, width, channels) interleaved samples, orientation applied."""
        L = self._L
        v = [ctypes.c_uint32() for _ in range(5)]
        L.jxlo_frame_info(self._h, idx, *[ctypes.byref(x) for x in v])
        w, h, nch, _, _ = [x.value for x in v]
        if (orientation or self.orientation) >= 5:
            w, h = h, w
        st = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2}[np.dtype(dtype)]
        out = np.empty((h, w, L.jxlo_frame_stream_channels(self._h, idx)), dtype=dtype)
        n = L.jxlo_frame_write_to_buffer(self._h, idx, st, orientation, out.ctypes.data)
        assert n == out.size
        return out

    def stage(self, name, dtype=np.float32):
        L = self._L
        w, h = ctypes.c_uint32(), ctypes.c_uint32()
        n = L.jxlo_stage(self._h, name.encode(), -1, ctypes.byref(w), ctypes.byref(h), None)
        planes = []
        for i in range(n):
            L.jxlo_stage(self._h, name.encode(), i, ctypes.byref(w), ctypes.byref(h), None)
            buf = np.empty((h.value, w.value), dtype=np.uint32)
            L.jxlo_stage(self._h, name.encode(), i, ctypes.byref(w), ctypes.byref(h), buf.ctypes.data)
            planes.append(buf.view(dtype))
        return planes

    def close(self):
        if self._h:
            self._L.jxlo_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def zstd_decompress(data: bytes) -> bytes:
    z = ctypes.CDLL("libzstd.so.1")
    z.ZSTD_getFrameContentSize.restype = ctypes.c_ulonglong
    z.ZSTD_getFrameContentSize.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    z.ZSTD_decompress.restype = ctypes.c_size_t
    z.ZSTD_decompress.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
    n = z.ZSTD_getFrameContentSize(data, len(data))
    if n >= (1 << 62):  # unknown size: streaming API
        z.ZSTD_createDStream.restype = ctypes.c_void_p
        z.ZSTD_decompressStream.restype = ctypes.c_size_t

        class Buf(ctypes.Structure):
            _fields_ = [("p", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]
        z.ZSTD_decompressStream.argtypes = [ctypes.c_void_p, ctypes.POINTER(Buf), ctypes.POINTER(Buf)]
        ds = z.ZSTD_createDStream()
        src = ctypes.create_string_buffer(data, len(data))
        ib = Buf(ctypes.cast(src, ctypes.c_void_p), len(data), 0)
        out = bytearray()
        chunk = ctypes.create_string_buffer(1 << 20)
        while ib.pos < ib.size:
            ob = Buf(ctypes.cast(chunk, ctypes.c_void_p), len(chunk), 0)
            r = z.ZSTD_decompressStream(ds, ctypes.byref(ob), ctypes.byref(ib))
            out += chunk.raw[:ob.pos]
            if r == 0 and ib.pos >= ib.size:
                break
        return bytes(out)
    out = ctypes.create_string_buffer(n)
    r = z.ZSTD_decompress(out, n, data, len(data))
    return out.raw[:r]
