"""ctypes wrapper around the JPEG-reconstruction oracle (oracle/jbr.mk -> oracle/_build/libjxlojbr.so) and the host
emulation of the device scan encoder (tests/emu/jpeg.mk -> tests/emu/_build/libjxlejpeg.so). Test infrastructure only."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIBS = {}


class JbrError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"JPEG reconstruction failed ({code}): {msg}")
        self.code = code


def _lib(emu):
    """Built through make every first use in a process: the recipes track the shared host code and kernel headers."""
    if emu not in _LIBS:
        d, mk, so = (("tests/emu", "jpeg.mk", "libjxlejpeg.so") if emu else ("oracle", "jbr.mk", "libjxlojbr.so"))
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, d), "-f", mk])
        L = ctypes.CDLL(os.path.join(ROOT, d, "_build", so))
        sig = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)),
               ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.c_size_t]
        L.jxlo_reconstruct_jpeg.argtypes = sig
        if emu:
            L.jxle_reconstruct_jpeg.argtypes = sig
        L.jxlo_free_bytes.argtypes = [ctypes.c_void_p]
        L.jxlo_jpeg_reconstruction_status.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
        _LIBS[emu] = L
    return _LIBS[emu]


def build():
    _lib(False)
    _lib(True)


def reconstruct_jpeg(data: bytes, emu=False) -> bytes:
    """The original JPEG of a JPEG transcode: the oracle's scalar scan encoder, or (emu) the host build of the device one."""
    L = _lib(emu)
    fn = L.jxle_reconstruct_jpeg if emu else L.jxlo_reconstruct_jpeg
    out, n, err = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_size_t(), ctypes.create_string_buffer(512)
    rc = fn(data, len(data), ctypes.byref(out), ctypes.byref(n), err, 512)
    if rc != 0:
        raise JbrError(rc, err.value.decode())
    try:
        return ctypes.string_at(out, n.value)
    finally:
        L.jxlo_free_bytes(out)


def jpeg_reconstruction_status(data: bytes) -> int:
    """0 unavailable, 1 available, 2 invalid (the shared host code in csrc/host/jbrd.cc)."""
    return _lib(False).jxlo_jpeg_reconstruction_status(data, len(data))
