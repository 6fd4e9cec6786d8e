"""jxl_oxide_b200 — H100-native JPEG XL decode hot path behind jxl-oxide's JxlImage / render_frame() API.

Python host-side mirror of the reference's public interface for this path
(crates/jxl-oxide/src/lib.rs: JxlImage::builder().read(..), image.render_frame(k) -> Render,
Render::image_planar()). All sample-level work runs in hand-written sm_90a CUDA kernels inside
libjxlb200.so (C ABI: include/jxlb200.h); this module only marshals bytes and pointers.

There is no CPU fallback: importing works anywhere (so the C ABI can be inspected), but creating a
decoder without a CUDA device raises JxlError.
"""
import ctypes
import os as _os

# One decoder context = one CUDA stream; give concurrent contexts their own hardware work queues
# (must be set before the CUDA context is created).
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libjxlb200.so")

OK, ERR_BITSTREAM, ERR_UNSUPPORTED, ERR_EOF, ERR_CUDA, ERR_INVALID_ARG, ERR_DEVICE_DECODE, ERR_OUT_OF_MEMORY = range(8)

# every symbol include/jxlb200.h declares
EXPORTED_SYMBOLS = [
    "jxlb_decoder_create", "jxlb_decoder_create_ex", "jxlb_decode_frame_sections", "jxlb_upsample", "jxlb_decoder_destroy",
    "jxlb_decode_hf_groups", "jxlb_dequant_idct", "jxlb_modular_decode_groups", "jxlb_last_error", "jxlb_decode", "jxlb_preload", "jxlb_decode_slot",
    "jxlb_image_get_info", "jxlb_image_original_icc",
    "jxlb_num_frames", "jxlb_frame_get_info", "jxlb_frame_channel_to_host", "jxlb_frame_stream_channels", "jxlb_frame_write_to_buffer", "jxlb_frame_write_to_device", "jxlb_frame_channel_device",
    "jxlb_release_frames", "jxlb_sync", "jxlb_launch_count", "jxlb_set_profile", "jxlb_profile_get",
    "jxlb_profile_reset", "jxlb_timeline_get", "jxlb_set_capture", "jxlb_set_fuse_filters", "jxlb_set_hf_streams_per_cta", "jxlb_set_hf_streams_per_warp", "jxlb_stage_count", "jxlb_stage_get",
    "jxlb_gaborish", "jxlb_epf", "jxlb_xyb_to_rgb", "jxlb_squeeze_inverse", "jxlb_rct_inverse", "jxlb_blend",
    "jxlb_pipeline_create", "jxlb_pipeline_destroy", "jxlb_pipeline_last_error", "jxlb_pipeline_preload", "jxlb_pipeline_submit",
    "jxlb_pipeline_wait", "jxlb_pipeline_release_output", "jxlb_pipeline_launch_count", "jxlb_pipeline_workers", "jxlb_pipeline_decoder",
    "jxlb_jpeg_reconstruction_status", "jxlb_reconstruct_jpeg", "jxlb_jpeg_copy",
    "jxlb_image_keyframes", "jxlb_decode_keyframe", "jxlb_pipeline_submit_keyframes", "jxlb_pipeline_wait_keyframe",
    "jxlb_frame_write_size", "jxlb_frame_write_ex", "jxlb_pipeline_submit_ex", "jxlb_pipeline_submit_keyframes_ex",
]

# Output layouts of Decoder.frame_write / jxlb_write_spec: Render::stream(), stream_no_alpha(), image_all_channels(),
# image_planar() (oriented)
LAYOUT_STREAM, LAYOUT_STREAM_NO_ALPHA, LAYOUT_ALL_INTERLEAVED, LAYOUT_ALL_PLANAR = range(4)
_LAYOUT_NAMES = {"stream": LAYOUT_STREAM, "stream_no_alpha": LAYOUT_STREAM_NO_ALPHA, "all_channels": LAYOUT_ALL_INTERLEAVED,
                 "planar": LAYOUT_ALL_PLANAR}
_SAMPLE_TYPES = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2}


class JxlError(RuntimeError):
    """Mirrors jxl_oxide's Result error values (decode errors are values, not crashes)."""

    def __init__(self, code, message):
        super().__init__(f"[{code}] {message}")
        self.code = code
        self.message = message

    @property
    def unsupported(self):
        return self.code == ERR_UNSUPPORTED


class _Options(ctypes.Structure):
    _fields_ = [("output_colour", ctypes.c_int32), ("max_frames", ctypes.c_uint32)]


class _FrameInfo(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint32) for n in ("width", "height", "num_channels", "num_color", "is_vardct", "duration")]


class _ImageInfo(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint32) for n in
                ("width", "height", "bits_per_sample", "num_extra_channels", "xyb_encoded", "grayscale", "orientation")]


class _Section(ctypes.Structure):
    _fields_ = [("data", ctypes.c_char_p), ("size", ctypes.c_size_t)]


class WriteSpec(ctypes.Structure):
    """jxlb_write_spec: what Decoder.frame_write and Pipeline.submit(spec=...) write."""
    _fields_ = [(n, ctypes.c_int32) for n in ("layout", "sample_type", "orientation", "render_spot_colour")]


def write_spec(layout=LAYOUT_STREAM, dtype=np.uint8, orientation=0, spot_colours=True):
    """A WriteSpec: `layout` a LAYOUT_* value or its name ("stream", "stream_no_alpha", "all_channels", "planar"), `dtype`
    uint8 / uint16 / float32, `orientation` 1..8 or 0 for the image's, `spot_colours` False to leave spot colours unmixed."""
    layout = _LAYOUT_NAMES.get(layout, layout)
    return WriteSpec(int(layout), _SAMPLE_TYPES[np.dtype(dtype)], int(orientation), int(bool(spot_colours)))


class _PipelineConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("workers", "heavy_frames", "hf_streams_per_cta", "no_affinity", "batch_streams")]


class EpfParams(ctypes.Structure):
    _fields_ = [("iters", ctypes.c_uint32), ("channel_scale", ctypes.c_float * 3), ("pass0_sigma_scale", ctypes.c_float),
                ("pass2_sigma_scale", ctypes.c_float), ("border_sad_mul", ctypes.c_float),
                ("sigma_for_modular", ctypes.c_float)]


_lib = None


def load_library():
    """Loads libjxlb200.so; fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise JxlError(ERR_CUDA, f"{LIB_PATH} is missing: build it with `python -m jxl_oxide_b200.build` "
                                 "(there is no CPU fallback)")
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, u32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint32
    L.jxlb_decoder_create.argtypes = [i32, ctypes.POINTER(vp)]
    L.jxlb_decoder_create.restype = i32
    L.jxlb_decoder_create_ex.argtypes = [i32, ctypes.c_uint64, ctypes.POINTER(vp)]
    L.jxlb_decoder_create_ex.restype = i32
    L.jxlb_decode_frame_sections.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(_Section), ctypes.c_size_t, ctypes.POINTER(_Options)]
    L.jxlb_upsample.argtypes = [vp, vp, u32, u32, u32, u32, vp, u32]
    L.jxlb_decode_hf_groups.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), u32, ctypes.POINTER(u32), ctypes.POINTER(u32)]
    L.jxlb_dequant_idct.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), u32, ctypes.POINTER(u32), ctypes.POINTER(u32)]
    L.jxlb_modular_decode_groups.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(vp), u32, u32, ctypes.POINTER(u32),
                                             ctypes.POINTER(u32), u32]
    L.jxlb_decoder_destroy.argtypes = [vp]
    L.jxlb_decoder_destroy.restype = None
    L.jxlb_last_error.argtypes = [vp]
    L.jxlb_last_error.restype = ctypes.c_char_p
    L.jxlb_decode.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(_Options)]
    L.jxlb_decode.restype = i32
    L.jxlb_preload.argtypes = [vp, i32, ctypes.c_char_p, ctypes.c_size_t]
    L.jxlb_decode_slot.argtypes = [vp, i32, ctypes.POINTER(_Options)]
    L.jxlb_image_get_info.argtypes = [vp, ctypes.POINTER(_ImageInfo)]
    L.jxlb_num_frames.argtypes = [vp]
    L.jxlb_frame_get_info.argtypes = [vp, i32, ctypes.POINTER(_FrameInfo)]
    L.jxlb_frame_channel_to_host.argtypes = [vp, i32, i32, vp, ctypes.c_size_t]
    L.jxlb_frame_write_to_buffer.argtypes = [vp, i32, i32, i32, vp, ctypes.c_size_t]
    L.jxlb_frame_write_to_device.argtypes = [vp, i32, i32, i32, vp, ctypes.c_size_t]
    L.jxlb_image_original_icc.argtypes = [vp, vp, ctypes.c_size_t]
    L.jxlb_image_original_icc.restype = ctypes.c_int64
    L.jxlb_frame_stream_channels.argtypes = [vp, i32]
    L.jxlb_frame_stream_channels.restype = i32
    L.jxlb_frame_channel_device.argtypes = [vp, i32, i32, ctypes.POINTER(vp), ctypes.POINTER(u32)]
    L.jxlb_release_frames.argtypes = [vp]
    L.jxlb_sync.argtypes = [vp]
    L.jxlb_launch_count.argtypes = [vp]
    L.jxlb_launch_count.restype = ctypes.c_uint64
    L.jxlb_set_capture.argtypes = [vp, i32]
    L.jxlb_set_fuse_filters.argtypes = [vp, i32]
    L.jxlb_set_hf_streams_per_cta.argtypes = [vp, i32]
    L.jxlb_set_hf_streams_per_warp.argtypes = [vp, i32]
    L.jxlb_set_profile.argtypes = [vp, i32]
    L.jxlb_profile_get.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_double)]
    L.jxlb_profile_reset.argtypes = [vp]
    L.jxlb_timeline_get.argtypes = [vp, i32, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]
    L.jxlb_stage_count.argtypes = [vp, ctypes.c_char_p]
    L.jxlb_stage_get.argtypes = [vp, ctypes.c_char_p, i32, ctypes.POINTER(u32), ctypes.POINTER(u32), vp]
    L.jxlb_blend.argtypes = [vp, vp, vp, vp, vp, u32, u32, u32, i32, i32, i32, i32]
    L.jxlb_gaborish.argtypes = [vp, ctypes.POINTER(vp), u32, u32, u32, ctypes.POINTER(ctypes.c_float)]
    L.jxlb_epf.argtypes = [vp, ctypes.POINTER(vp), u32, u32, u32, vp, u32, ctypes.POINTER(EpfParams)]
    L.jxlb_xyb_to_rgb.argtypes = [vp, ctypes.POINTER(vp), u32, u32, u32, ctypes.POINTER(ctypes.c_float),
                                  ctypes.POINTER(ctypes.c_float), ctypes.c_float, i32]
    L.jxlb_squeeze_inverse.argtypes = [vp, vp, u32, u32, u32, vp, u32, u32, u32, vp, u32, i32]
    L.jxlb_rct_inverse.argtypes = [vp, ctypes.POINTER(vp), u32, u32, u32, u32]
    L.jxlb_pipeline_create.argtypes = [i32, ctypes.POINTER(_PipelineConfig), ctypes.POINTER(vp)]
    L.jxlb_pipeline_destroy.argtypes = [vp]
    L.jxlb_pipeline_destroy.restype = None
    L.jxlb_pipeline_last_error.argtypes = [vp]
    L.jxlb_pipeline_last_error.restype = ctypes.c_char_p
    L.jxlb_pipeline_preload.argtypes = [vp, i32, ctypes.c_char_p, ctypes.c_size_t]
    L.jxlb_pipeline_submit.argtypes = [vp, vp, ctypes.c_size_t, i32, i32, vp, ctypes.c_size_t, ctypes.c_uint64]
    L.jxlb_pipeline_wait.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(i32), ctypes.POINTER(vp),
                                     ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.c_size_t]
    L.jxlb_pipeline_submit_keyframes.argtypes = [vp, vp, ctypes.c_size_t, i32, i32, vp, ctypes.c_size_t, ctypes.c_uint64]
    L.jxlb_pipeline_wait_keyframe.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(i32), ctypes.POINTER(i32),
                                              ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.c_size_t]
    L.jxlb_pipeline_release_output.argtypes = [vp, vp]
    L.jxlb_pipeline_launch_count.argtypes = [vp]
    L.jxlb_pipeline_launch_count.restype = ctypes.c_uint64
    L.jxlb_pipeline_workers.argtypes = [vp]
    L.jxlb_pipeline_decoder.argtypes = [vp, i32]
    L.jxlb_pipeline_decoder.restype = vp
    L.jxlb_jpeg_reconstruction_status.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    L.jxlb_jpeg_reconstruction_status.restype = i32
    L.jxlb_reconstruct_jpeg.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
    L.jxlb_reconstruct_jpeg.restype = i32
    L.jxlb_jpeg_copy.argtypes = [vp, vp, ctypes.c_size_t]
    L.jxlb_jpeg_copy.restype = i32
    L.jxlb_image_keyframes.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(i32), ctypes.POINTER(i32)]
    L.jxlb_image_keyframes.restype = i32
    L.jxlb_decode_keyframe.argtypes = [vp, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(_Options), i32]
    L.jxlb_frame_write_size.argtypes = [vp, i32, ctypes.POINTER(WriteSpec), ctypes.POINTER(u32), ctypes.POINTER(ctypes.c_uint64)]
    L.jxlb_frame_write_size.restype = i32
    L.jxlb_frame_write_ex.argtypes = [vp, i32, ctypes.POINTER(WriteSpec), vp, ctypes.c_size_t, i32]
    L.jxlb_frame_write_ex.restype = i32
    L.jxlb_pipeline_submit_ex.argtypes = [vp, vp, ctypes.c_size_t, i32, ctypes.POINTER(WriteSpec), vp, ctypes.c_size_t, i32, ctypes.c_uint64]
    L.jxlb_pipeline_submit_keyframes_ex.argtypes = [vp, vp, ctypes.c_size_t, i32, ctypes.POINTER(WriteSpec), vp, ctypes.c_size_t, i32,
                                                    ctypes.c_uint64]
    _lib = L
    return L


class Decoder:
    """One decoder = one CUDA stream + its HBM planes (RenderContext analogue)."""

    def __init__(self, device=0, mem_limit=0):
        """`mem_limit`: allocation budget in bytes of HBM (0 = unlimited), AllocTracker::with_limit's counterpart."""
        L = load_library()
        h = ctypes.c_void_p()
        rc = L.jxlb_decoder_create_ex(device, int(mem_limit), ctypes.byref(h))
        if rc != OK:
            raise JxlError(rc, "cannot create CUDA decoder (no CUDA device? this path has no CPU fallback)")
        self._h = h
        self._L = L
        self.device = int(device)

    def _check(self, rc):
        if rc != OK:
            raise JxlError(rc, self._L.jxlb_last_error(self._h).decode(errors="replace"))

    def decode(self, data: bytes, output_colour=0, max_frames=0):
        opt = _Options(output_colour, max_frames)
        self._check(self._L.jxlb_decode(self._h, data, len(data), ctypes.byref(opt)))

    def decode_sections(self, header: bytes, sections, output_colour=0, max_frames=0):
        """jxlb_decode_frame_sections: `header` = signature .. TOC, `sections` = the TOC entries' bytes in bitstream order."""
        arr = (_Section * len(sections))(*[_Section(s, len(s)) for s in sections])
        opt = _Options(output_colour, max_frames)
        self._check(self._L.jxlb_decode_frame_sections(self._h, header, len(header), arr, len(sections), ctypes.byref(opt)))

    def reconstruct_jpeg(self, data: bytes) -> bytes:
        """JxlImage::reconstruct_jpeg: the original JPEG file of a JPEG transcode (a `jbrd` box), scans encoded on the GPU.
        Releases this decoder's frames. JxlError UNSUPPORTED when the file has no reconstruction data."""
        n = ctypes.c_size_t()
        self._check(self._L.jxlb_reconstruct_jpeg(self._h, data, len(data), ctypes.byref(n)))
        buf = ctypes.create_string_buffer(max(n.value, 1))
        self._check(self._L.jxlb_jpeg_copy(self._h, buf, n.value))
        return buf.raw[:n.value]

    def _stage_planes(self, fn, data, dtype):
        import torch
        w, h = ctypes.c_uint32(), ctypes.c_uint32()
        self._check(fn(self._h, data, len(data), None, 0, ctypes.byref(w), ctypes.byref(h)))
        planes = [torch.empty((h.value, w.value), dtype=dtype, device=f"cuda:{self.device}") for _ in range(3)]
        ptrs = (ctypes.c_void_p * 3)(*[int(p.data_ptr()) for p in planes])
        self._check(fn(self._h, data, len(data), ptrs, w.value, ctypes.byref(w), ctypes.byref(h)))
        return planes

    def decode_hf_groups(self, data):
        """jxlb_decode_hf_groups: the quantised HF coefficients (X, Y, B; int32 CUDA tensors)."""
        import torch
        return self._stage_planes(self._L.jxlb_decode_hf_groups, data, torch.int32)

    def dequant_idct(self, data):
        """jxlb_dequant_idct: the XYB samples after dequantisation and the inverse transforms (float32 CUDA tensors)."""
        import torch
        return self._stage_planes(self._L.jxlb_dequant_idct, data, torch.float32)

    def modular_decode_groups(self, data):
        """jxlb_modular_decode_groups: the coded channels of the frame's Modular image before the inverse transforms."""
        import torch
        n = ctypes.c_uint32()
        dims = (ctypes.c_uint32 * 2048)()
        self._check(self._L.jxlb_modular_decode_groups(self._h, data, len(data), None, 0, 0, ctypes.byref(n), dims, 2048))
        shapes = [(dims[2 * i + 1], dims[2 * i]) for i in range(n.value)]
        stride = max([s[1] for s in shapes] + [1])
        chans = [torch.empty((max(s[0], 1), stride), dtype=torch.int32, device=f"cuda:{self.device}") for s in shapes]
        ptrs = (ctypes.c_void_p * len(chans))(*[int(c.data_ptr()) for c in chans])
        self._check(self._L.jxlb_modular_decode_groups(self._h, data, len(data), ptrs, len(chans), stride, ctypes.byref(n), dims, 2048))
        return [c[: s[0], : s[1]] for c, s in zip(chans, shapes)]

    def upsample(self, src, factor):
        """features::upsample with the default weights on a device tensor (h, w) float32 -> (h * factor, w * factor)."""
        import torch
        h, w = src.shape
        out = torch.empty((h * factor, w * factor), dtype=torch.float32, device=src.device)
        self._check(self._L.jxlb_upsample(self._h, int(src.data_ptr()), w, h, src.stride(0), factor, int(out.data_ptr()), out.stride(0)))
        return out

    def decode_keyframe(self, data: bytes, keyframe, output_colour=0):
        """jxlb_decode_keyframe (JxlImage::render_frame(k)): keyframe `keyframe` alone, resident as frame 0. Only the
        segment that holds it is decoded, and only one keyframe is resident at a time."""
        opt = _Options(output_colour, 0)
        self._check(self._L.jxlb_decode_keyframe(self._h, data, len(data), ctypes.byref(opt), int(keyframe)))

    def preload(self, slot, data: bytes):
        self._check(self._L.jxlb_preload(self._h, slot, data, len(data)))

    def decode_slot(self, slot, output_colour=0, max_frames=0):
        opt = _Options(output_colour, max_frames)
        self._check(self._L.jxlb_decode_slot(self._h, slot, ctypes.byref(opt)))

    def image_info(self):
        info = _ImageInfo()
        self._check(self._L.jxlb_image_get_info(self._h, ctypes.byref(info)))
        return info

    def num_frames(self):
        return self._L.jxlb_num_frames(self._h)

    def frame_info(self, frame):
        info = _FrameInfo()
        self._check(self._L.jxlb_frame_get_info(self._h, frame, ctypes.byref(info)))
        return info

    def frame_planar(self, frame):
        """numpy (channels, height, width) float32 — Render::image_planar()."""
        info = self.frame_info(frame)
        out = np.empty((info.num_channels, info.height, info.width), dtype=np.float32)
        for c in range(info.num_channels):
            self._check(self._L.jxlb_frame_channel_to_host(self._h, frame, c, out[c].ctypes.data, info.width))
        return out

    def frame_channel_device(self, frame, channel):
        ptr, stride = ctypes.c_void_p(), ctypes.c_uint32()
        self._check(self._L.jxlb_frame_channel_device(self._h, frame, channel, ctypes.byref(ptr), ctypes.byref(stride)))
        return ptr.value, stride.value

    def release_frames(self):
        self._check(self._L.jxlb_release_frames(self._h))

    def sync(self):
        self._check(self._L.jxlb_sync(self._h))

    def launch_count(self):
        return int(self._L.jxlb_launch_count(self._h))

    def set_profile(self, on=True):
        self._L.jxlb_set_profile(self._h, int(on))

    def profile(self, name):
        """(launches, total_ms) of a kernel family, timed with CUDA events on the decoder's stream."""
        n, ms = ctypes.c_uint64(), ctypes.c_double()
        self._check(self._L.jxlb_profile_get(self._h, name.encode(), ctypes.byref(n), ctypes.byref(ms)))
        return n.value, ms.value

    def profile_reset(self):
        self._check(self._L.jxlb_profile_reset(self._h))

    def frame_to_host(self, frame, out):
        """Copies all channels of a frame into a preallocated (channels, h, w) float32 array."""
        for c in range(out.shape[0]):
            self._check(self._L.jxlb_frame_channel_to_host(self._h, frame, c, out[c].ctypes.data, out.shape[2]))

    def original_icc(self):
        """JxlImage::original_icc: the embedded ICC profile's bytes (b"" when the image has none)."""
        n = self._L.jxlb_image_original_icc(self._h, None, 0)
        if n <= 0:
            return b""
        buf = ctypes.create_string_buffer(n)
        self._L.jxlb_image_original_icc(self._h, buf, n)
        return buf.raw

    def frame_to_buffer(self, frame, dtype=np.uint8, orientation=0, out=None):
        """ImageStream::write_to_buffer: (height, width, channels) interleaved u8 / u16 / f32 samples with the
        orientation applied (0 = the image header's). `out`: a C-contiguous array of that shape to fill (e.g. pinned)."""
        spec = write_spec(LAYOUT_STREAM, dtype, orientation)
        out, dst, nbytes = self._write_target(frame, spec, out, on_device=False)
        self._check(self._L.jxlb_frame_write_to_buffer(self._h, frame, spec.sample_type, spec.orientation, dst, nbytes))
        return out

    def frame_to_torch(self, frame, dtype=np.uint8, orientation=0, out=None):
        """frame_to_buffer() with the packed (height, width, channels) samples left in HBM as a torch tensor on this
        decoder's GPU (jxlb_frame_write_to_device); torch only owns the memory."""
        spec = write_spec(LAYOUT_STREAM, dtype, orientation)
        out, dst, nbytes = self._write_target(frame, spec, out, on_device=True)
        self._check(self._L.jxlb_frame_write_to_device(self._h, frame, spec.sample_type, spec.orientation, dst, nbytes))
        return out

    def frame_write_shape(self, frame, spec: WriteSpec):
        """(shape, nbytes) of frame_write's output: (height, width, channels) interleaved or (channels, height, width)
        planar, oriented."""
        n, nbytes = ctypes.c_uint32(), ctypes.c_uint64()
        self._check(self._L.jxlb_frame_write_size(self._h, frame, ctypes.byref(spec), ctypes.byref(n), ctypes.byref(nbytes)))
        info = self.frame_info(frame)
        orient = spec.orientation or self.image_info().orientation
        w, h = (info.height, info.width) if orient >= 5 else (info.width, info.height)
        shape = (n.value, h, w) if spec.layout == LAYOUT_ALL_PLANAR else (h, w, n.value)
        return shape, nbytes.value

    def _write_target(self, frame, spec: WriteSpec, out, on_device):
        """(out, pointer, nbytes) of a write of `frame` as `spec` asks: `out` checked against frame_write_shape(), or
        allocated when None: a numpy array, or with on_device a torch tensor on this decoder's GPU."""
        shape, nbytes = self.frame_write_shape(frame, spec)
        if on_device:
            import torch
            tdt = {0: torch.uint8, 1: torch.uint16, 2: torch.float32}[spec.sample_type]
            if out is None:
                out = torch.empty(shape, dtype=tdt, device=f"cuda:{self.device}")
            if tuple(out.shape) != shape or out.dtype != tdt or not out.is_contiguous() or not out.is_cuda:
                raise ValueError(f"out must be a contiguous CUDA {tdt} tensor of shape {shape}")
            return out, out.data_ptr(), nbytes
        dtype = {0: np.uint8, 1: np.uint16, 2: np.float32}[spec.sample_type]
        if out is None:
            out = np.empty(shape, dtype=dtype)
        if out.shape != shape or out.dtype != np.dtype(dtype) or not out.flags.c_contiguous:
            raise ValueError(f"out must be a C-contiguous {np.dtype(dtype)} array of shape {shape}")
        return out, out.ctypes.data, nbytes

    def frame_write(self, frame, layout=LAYOUT_STREAM, dtype=np.uint8, orientation=0, spot_colours=True, out=None):
        """One of the Render layouts (jxlb_frame_write_ex), packed on the device: `layout` as for write_spec(). Returns a
        numpy array, or fills `out`: a C-contiguous numpy array, or a contiguous torch CUDA tensor of this decoder's GPU
        (the samples then stay in HBM), of frame_write_shape()'s shape and `dtype`."""
        spec = write_spec(layout, dtype, orientation, spot_colours)
        on_device = hasattr(out, "data_ptr")
        out, dst, nbytes = self._write_target(frame, spec, out, on_device)
        self._check(self._L.jxlb_frame_write_ex(self._h, frame, ctypes.byref(spec), dst, nbytes, int(on_device)))
        return out

    def set_capture(self, on=True):
        self._L.jxlb_set_capture(self._h, int(on))

    def timeline(self):
        """[(name, t0_ms, t1_ms)] of the profiled launches / host phases since profile_reset()."""
        n = self._L.jxlb_timeline_get(self._h, -1, None, 0, None, None)
        out = []
        buf = ctypes.create_string_buffer(64)
        t0, t1 = ctypes.c_double(), ctypes.c_double()
        for i in range(max(n, 0)):
            self._L.jxlb_timeline_get(self._h, i, buf, 64, ctypes.byref(t0), ctypes.byref(t1))
            out.append((buf.value.decode(), t0.value, t1.value))
        return out

    def set_fuse_filters(self, on=True):
        self._L.jxlb_set_fuse_filters(self._h, int(on))

    def set_hf_streams_per_cta(self, streams):
        """HF streams per CTA: 0 (default, = 16), 4 (= 8), 8, 16, 32: one warp per stream; 64 / 128: one thread per stream."""
        if self._L.jxlb_set_hf_streams_per_cta(self._h, int(streams)) != 0:
            raise ValueError("streams per CTA must be 0, 4, 8, 16, 32, 64 or 128")

    def set_hf_streams_per_warp(self, streams):
        """Thread-per-stream HF schedules: streams per warp, 0 (default), 4, 8, 16 or 32 (jxlb_set_hf_streams_per_warp)."""
        if self._L.jxlb_set_hf_streams_per_warp(self._h, int(streams)) != 0:
            raise ValueError("streams per warp must be 0, 4, 8, 16 or 32")

    def stage(self, name, dtype=np.float32):
        n = self._L.jxlb_stage_count(self._h, name.encode())
        planes = []
        for i in range(n):
            w, h = ctypes.c_uint32(), ctypes.c_uint32()
            self._check(self._L.jxlb_stage_get(self._h, name.encode(), i, ctypes.byref(w), ctypes.byref(h), None))
            buf = np.empty((h.value, w.value), dtype=np.uint32)
            self._check(self._L.jxlb_stage_get(self._h, name.encode(), i, ctypes.byref(w), ctypes.byref(h), buf.ctypes.data))
            planes.append(buf.view(dtype))
        return planes

    # ---- stage-level entry points on device memory (torch tensors) ----
    def _plane_ptrs(self, planes):
        arr = (ctypes.c_void_p * 3)(*[int(p.data_ptr()) for p in planes])
        return arr

    def gaborish(self, planes, weights):
        h, w = planes[0].shape
        wts = (ctypes.c_float * 6)(*[float(x) for row in weights for x in row])
        self._check(self._L.jxlb_gaborish(self._h, self._plane_ptrs(planes), w, h, planes[0].stride(0), wts))

    def epf(self, planes, sigma, params: EpfParams):
        h, w = planes[0].shape
        sp = int(sigma.data_ptr()) if sigma is not None else None
        ss = sigma.stride(0) if sigma is not None else 0
        self._check(self._L.jxlb_epf(self._h, self._plane_ptrs(planes), w, h, planes[0].stride(0), sp, ss, ctypes.byref(params)))

    def xyb_to_rgb(self, planes, opsin_bias, inv_matrix, intensity_target=255.0, srgb_tf=True):
        h, w = planes[0].shape
        ob = (ctypes.c_float * 3)(*opsin_bias)
        m = (ctypes.c_float * 9)(*inv_matrix)
        self._check(self._L.jxlb_xyb_to_rgb(self._h, self._plane_ptrs(planes), w, h, planes[0].stride(0), ob, m,
                                            float(intensity_target), int(srgb_tf)))

    def squeeze_inverse(self, avg, res, out, horizontal):
        self._check(self._L.jxlb_squeeze_inverse(self._h, int(avg.data_ptr()), avg.shape[1], avg.shape[0], avg.stride(0),
                                                 int(res.data_ptr()), res.shape[1], res.shape[0], max(res.stride(0), 1),
                                                 int(out.data_ptr()), out.stride(0), int(horizontal)))

    def blend(self, base, patch, base_alpha, new_alpha, mode, clamp=False, premultiplied=False, swapped=False):
        """blend_single on equally shaped device tensors, in place on `base` (alpha tensors may be None)."""
        h, w = base.shape
        ptr = lambda t: int(t.data_ptr()) if t is not None else None
        self._check(self._L.jxlb_blend(self._h, ptr(base), ptr(patch), ptr(base_alpha), ptr(new_alpha), w, h, base.stride(0),
                                       int(mode), int(clamp), int(premultiplied), int(swapped)))

    def rct_inverse(self, planes, rct_type):
        h, w = planes[0].shape
        self._check(self._L.jxlb_rct_inverse(self._h, self._plane_ptrs(planes), w, h, planes[0].stride(0), rct_type))

    def close(self):
        if getattr(self, "_h", None):
            if getattr(self, "_owned", True):
                self._L.jxlb_decoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Pipeline:
    """Many independent frames through one GPU (jxlb_pipeline_*): `workers` decoder contexts fed from one queue, at
    most `heavy_frames` of them past the LF stage. The analogue of decoding keyframes in a rayon par_iter
    (crates/jxl-oxide-cli/src/decode.rs:285-320)."""

    OUT_NONE, OUT_PLANAR_F32, OUT_U8, OUT_U16, OUT_U8_DEVICE, OUT_U16_DEVICE = 0, 1, 2, 3, 4, 5

    def __init__(self, device=0, workers=0, heavy_frames=0, hf_streams_per_cta=0, no_affinity=False, batch_streams=0):
        self._L = load_library()
        self.device = device
        cfg = _PipelineConfig(int(workers), int(heavy_frames), int(hf_streams_per_cta), int(bool(no_affinity)), int(batch_streams))
        h = ctypes.c_void_p()
        rc = self._L.jxlb_pipeline_create(device, ctypes.byref(cfg), ctypes.byref(h))
        if rc != OK:
            raise JxlError(rc, "cannot create a pipeline (no CUDA device? there is no CPU fallback)")
        self._h = h
        self._keep = {}      # tag -> objects that must outlive the job (input bytes, output arrays)
        self._reports = {}   # tag of a keyframe submission -> reports still to come
        self._slot_reports = {}  # preloaded slot -> reports a keyframe submission of it gives
        self._next_tag = 0
        self.in_flight = 0

    def _err(self, rc):
        raise JxlError(rc, (self._L.jxlb_pipeline_last_error(self._h) or b"").decode())

    def preload(self, slot, data: bytes):
        rc = self._L.jxlb_pipeline_preload(self._h, slot, data, len(data))
        if rc != OK:
            self._err(rc)
        self._slot_reports[slot] = _keyframe_reports(data)

    def _take(self, tag):
        """The objects kept for `tag`, released with its last report."""
        left = self._reports.get(tag, 1) - 1
        if left > 0:
            self._reports[tag] = left
            return self._keep.get(tag)
        self._reports.pop(tag, None)
        return self._keep.pop(tag, None)

    @classmethod
    def _dst(cls, out, mode):
        if mode is None and not hasattr(out, "data_ptr"):  # out=None + explicit mode: pixels in a pipeline-owned pinned buffer
            mode = cls.OUT_NONE if out is None else {np.dtype(np.float32): 1, np.dtype(np.uint8): 2, np.dtype(np.uint16): 3}[out.dtype]
        if out is not None and hasattr(out, "data_ptr"):  # a torch CUDA tensor: packed on the device, never leaves HBM
            if mode is None or mode < 4:
                mode = {1: cls.OUT_U8_DEVICE, 2: cls.OUT_U16_DEVICE}[out.element_size()]
            dst, nbytes = int(out.data_ptr()), out.numel() * out.element_size()
        else:
            dst, nbytes = (out.ctypes.data, out.nbytes) if out is not None else (None, 0)
        return mode, dst, nbytes

    @staticmethod
    def _spec_dst(out):
        """(dst, nbytes, on_device) of a spec submission: a torch CUDA tensor, a numpy array, or None for the ring."""
        if out is None:
            return None, 0, 0
        if hasattr(out, "data_ptr"):
            return int(out.data_ptr()), out.numel() * out.element_size(), 1
        return out.ctypes.data, out.nbytes, 0

    def submit(self, data=None, slot=-1, out=None, mode=None, tag=None, spec=None):
        """Queues one frame: `data` (bytes) or a preloaded `slot`. `out`: None (decode only), a float32 (c, h, w) array
        (planar) or a uint8 / uint16 (h, w, c) array (interleaved); it must stay untouched until wait() reports the tag.
        With `spec` (a WriteSpec, see write_spec()) the frame is written as it describes, into `out` (a numpy array, or a
        torch CUDA tensor that is filled on the device) or, with out=None, into a buffer of the pipeline's ring."""
        if tag is None:
            tag = self._next_tag
            self._next_tag += 1
        buf = None
        if data is not None:
            buf = ctypes.c_char_p(data)
        src = ctypes.cast(buf, ctypes.c_void_p) if buf is not None else None
        if spec is not None:
            dst, nbytes, on_device = self._spec_dst(out)
            rc = self._L.jxlb_pipeline_submit_ex(self._h, src, len(data) if data is not None else 0, slot, ctypes.byref(spec), dst,
                                                 nbytes, on_device, tag)
        else:
            mode, dst, nbytes = self._dst(out, mode)
            rc = self._L.jxlb_pipeline_submit(self._h, src, len(data) if data is not None else 0, slot, mode, dst, nbytes, tag)
        if rc != OK:
            self._err(rc)
        self._keep[tag] = (data, buf, out)
        self.in_flight += 1
        return tag

    def wait(self, want_output=False):
        """Blocks until one frame has finished; returns its tag, or (tag, address, nbytes) of its pixels with
        want_output (a pipeline-owned pinned buffer must then go back through release_output()). Raises JxlError when
        that frame failed. Without want_output a pipeline-owned buffer is returned to the ring at once."""
        tag, status = ctypes.c_uint64(), ctypes.c_int32()
        out, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        msg = ctypes.create_string_buffer(256)
        rc = self._L.jxlb_pipeline_wait(self._h, ctypes.byref(tag), ctypes.byref(status), ctypes.byref(out), ctypes.byref(nbytes), msg, 256)
        if rc != OK:
            raise JxlError(rc, "no frame in flight")
        self.in_flight -= 1
        kept = self._take(tag.value)
        if status.value != OK:
            raise JxlError(status.value, msg.value.decode(errors="replace"))
        owned = out.value is not None and (kept is None or kept[2] is None)
        if kept is not None and kept[2] is not None and hasattr(kept[2], "data_ptr"):
            owned = False
        if want_output:
            return tag.value, out.value, nbytes.value
        if owned:
            self._L.jxlb_pipeline_release_output(self._h, out)
        return tag.value

    def submit_keyframes(self, data=None, slot=-1, out=None, mode=None, tag=None, spec=None):
        """Queues every keyframe of `data` (bytes) or of a preloaded `slot`, one task per independent segment
        (jxlb_pipeline_submit_keyframes). `out` as for submit() with a leading keyframe axis: (num_keyframes, ...);
        keyframe k lands in out[k]. Collect the reports with wait_keyframe(); with out=None and a mode or a spec, release
        each output as it is consumed. `spec` as for submit(). Returns the tag."""
        if tag is None:
            tag = self._next_tag
            self._next_tag += 1
        reports = _keyframe_reports(data) if data is not None else self._slot_reports.get(slot, 1)
        buf = ctypes.c_char_p(data) if data is not None else None
        src = ctypes.cast(buf, ctypes.c_void_p) if buf is not None else None
        if spec is not None:
            dst, nbytes, on_device = self._spec_dst(out)
            rc = self._L.jxlb_pipeline_submit_keyframes_ex(self._h, src, len(data) if data is not None else 0, slot, ctypes.byref(spec),
                                                           dst, nbytes, on_device, tag)
        else:
            mode, dst, nbytes = self._dst(out, mode)
            rc = self._L.jxlb_pipeline_submit_keyframes(self._h, src, len(data) if data is not None else 0, slot, mode, dst, nbytes, tag)
        if rc != OK:
            self._err(rc)
        if reports:
            self._keep[tag] = (data, buf, out)
            self._reports[tag] = reports
        self.in_flight += reports
        return tag

    def wait_keyframe(self, want_output=False):
        """Blocks until one keyframe (or frame of submit()) has finished; returns (tag, keyframe), or
        (tag, keyframe, address, nbytes) with want_output; keyframe is -1 for a frame of submit(). Raises JxlError, with
        the report's `tag` and `keyframe` attributes, when that keyframe failed."""
        tag, kf, status = ctypes.c_uint64(), ctypes.c_int32(), ctypes.c_int32()
        out, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        msg = ctypes.create_string_buffer(256)
        rc = self._L.jxlb_pipeline_wait_keyframe(self._h, ctypes.byref(tag), ctypes.byref(kf), ctypes.byref(status), ctypes.byref(out),
                                                 ctypes.byref(nbytes), msg, 256)
        if rc != OK:
            raise JxlError(rc, "no frame in flight")
        self.in_flight -= 1
        kept = self._take(tag.value)
        if status.value != OK:
            e = JxlError(status.value, msg.value.decode(errors="replace"))
            e.tag, e.keyframe = tag.value, kf.value
            raise e
        owned = out.value is not None and (kept is None or kept[2] is None)
        if want_output:
            return tag.value, kf.value, out.value, nbytes.value
        if owned:
            self._L.jxlb_pipeline_release_output(self._h, out)
        return tag.value, kf.value

    def release_output(self, address):
        self._L.jxlb_pipeline_release_output(self._h, ctypes.c_void_p(address))

    def drain(self):
        """Waits for every frame in flight; raises the first error after all have been collected."""
        first = None
        while self.in_flight:
            try:
                self.wait()
            except JxlError as e:
                first = first or e
        if first:
            raise first

    def launch_count(self):
        return int(self._L.jxlb_pipeline_launch_count(self._h))

    def workers(self):
        return int(self._L.jxlb_pipeline_workers(self._h))

    def decoder(self, index):
        """The index-th worker's Decoder (profiling knobs only; not owned by the returned object)."""
        h = self._L.jxlb_pipeline_decoder(self._h, index)
        if not h:
            raise IndexError(index)
        d = Decoder.__new__(Decoder)
        d._L = self._L
        d._h = ctypes.c_void_p(h)
        d._owned = False  # borrowed: destroyed with the pipeline
        d.device = self.device
        return d

    def close(self):
        if getattr(self, "_h", None):
            self._L.jxlb_pipeline_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Render:
    """Result of JxlImage.render_frame(): planar f32 channels (crates/jxl-oxide/src/lib.rs:1080-1216). The layouts with
    the orientation applied are packed on the device from the frame still resident in `decoder`."""

    def __init__(self, planar, num_color, is_vardct, decoder=None, frame=0, spot_colours=True):
        self._planar = planar
        self.num_color = num_color
        self.is_vardct = is_vardct
        self._dec = decoder
        self._frame = frame
        self._spot_colours = spot_colours

    def image_planar(self, oriented=False):
        """The stored planes (channels, height, width) float32; oriented=True: Render::image_planar(), every channel with
        the image's orientation applied."""
        if not oriented:
            return self._planar
        return self._dec.frame_write(self._frame, LAYOUT_ALL_PLANAR, np.float32)

    def stream(self, no_alpha=False, dtype=np.float32, out=None):
        """Render::stream() / stream_no_alpha() written out: colour, black and alpha channels (h, w, c), spot colours
        mixed in unless JxlImage.set_render_spot_color(False), oriented. `out` as for Decoder.frame_write()."""
        layout = LAYOUT_STREAM_NO_ALPHA if no_alpha else LAYOUT_STREAM
        return self._dec.frame_write(self._frame, layout, dtype, spot_colours=self._spot_colours, out=out)

    def image_all_channels(self, dtype=np.float32, out=None):
        """Render::image_all_channels(): every channel interleaved (h, w, c), oriented."""
        return self._dec.frame_write(self._frame, LAYOUT_ALL_INTERLEAVED, dtype, out=out)

    def color_channels(self):
        return self._planar[: self.num_color]

    def extra_channels(self):
        return self._planar[self.num_color:]


class JxlImage:
    """Mirror of jxl_oxide::JxlImage for the decode hot path."""

    def __init__(self, data: bytes, device=0, output_colour=0):
        self._data = bytes(data)
        self._jpeg_dec = None
        self._dec = Decoder(device)
        self._dec.decode(data, output_colour=output_colour)
        info = self._dec.image_info()
        self.width, self.height = info.width, info.height
        self.bits_per_sample = info.bits_per_sample
        self.num_extra_channels = info.num_extra_channels
        self.xyb_encoded = bool(info.xyb_encoded)
        self._grayscale = bool(info.grayscale)
        self._render_spot_color = True

    @classmethod
    def read(cls, data: bytes, **kw):
        return cls(data, **kw)

    @classmethod
    def open(cls, path, **kw):
        with open(path, "rb") as f:
            return cls(f.read(), **kw)

    def num_loaded_keyframes(self):
        return self._dec.num_frames()

    def render_frame(self, keyframe_index=0):
        info = self._dec.frame_info(keyframe_index)
        return Render(self._dec.frame_planar(keyframe_index), info.num_color, bool(info.is_vardct), self._dec, keyframe_index,
                      self._render_spot_color)

    def render_spot_color(self):
        return self._render_spot_color

    def set_render_spot_color(self, render_spot_color: bool):
        """JxlImage::set_render_spot_color (lib.rs:599-610): whether Render.stream() mixes the spot colours in. Turning it on
        for a grayscale image is ignored, as the reference does."""
        if render_spot_color and self._grayscale:
            return self
        self._render_spot_color = bool(render_spot_color)
        return self

    @property
    def decoder(self):
        return self._dec

    def jpeg_reconstruction_status(self):
        """0 unavailable (no jbrd box), 1 available, 2 invalid (JxlImage::jpeg_reconstruction_status)."""
        return jpeg_reconstruction_status(self._data)

    def reconstruct_jpeg(self) -> bytes:
        """The original JPEG file, rebuilt from the bytes this image was read from (on a decoder of its own, so the
        decoded frames stay available)."""
        if self._jpeg_dec is None:
            self._jpeg_dec = Decoder(self._dec.device)
        return self._jpeg_dec.reconstruct_jpeg(self._data)


def image_keyframes(data: bytes):
    """(num_keyframes, num_segments, status) from a header-only pass (jxlb_image_keyframes; no device needed). status is
    OK, or the error of a last frame that is malformed or cut off, which is then counted as one more keyframe; when
    not even the image header can be read, JxlError is raised."""
    nk, ns = ctypes.c_int32(), ctypes.c_int32()
    rc = load_library().jxlb_image_keyframes(data, len(data), ctypes.byref(nk), ctypes.byref(ns))
    if rc != OK and nk.value == 0:
        raise JxlError(rc, "cannot read the image header")
    return nk.value, ns.value, rc


def _keyframe_reports(data):
    """How many reports jxlb_pipeline_submit_keyframes gives for `data`: one per keyframe, or one for an unreadable header."""
    try:
        return image_keyframes(data)[0]
    except JxlError:
        return 1


def jpeg_reconstruction_status(data: bytes) -> int:
    """0 unavailable (no jbrd box), 1 available, 2 invalid; host-side parsing only, no device needed."""
    return int(load_library().jxlb_jpeg_reconstruction_status(data, len(data)))
