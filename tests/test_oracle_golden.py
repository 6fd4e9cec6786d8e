"""CPU tests: pin the oracle against the reference's own golden vectors (SURVEY.md §8c)."""
import ctypes
import math
import struct

import numpy as np
import pytest

from conftest import fixture_bytes

MODULAR_GOLDENS = ["grayalpha", "squeeze_edge", "issue_311"]


@pytest.mark.parametrize("name", MODULAR_GOLDENS)
def test_modular_golden_bit_exact(oracle, name):
    """crates/jxl-oxide-tests/tests/decode/mod.rs:29-86 with threshold 0 (8-bit modular is exact:
    v/255*65535+0.5 is injective)."""
    gold = oracle.zstd_decompress(fixture_bytes(name, "output.buf.zst"))
    w, h, ch = struct.unpack("<III", gold[:12])
    img = oracle.OracleImage(fixture_bytes(name, "input.jxl"))
    planes, _, is_vardct = img.frame(0)
    assert not is_vardct
    assert gold[12] == 0 and gold[-1] == 0xFF
    exp = np.frombuffer(gold, dtype="<u2", count=w * h * ch, offset=13).reshape(ch, h, w)
    act = (planes * np.float32(65535.0) + np.float32(0.5)).astype(np.uint16)
    assert planes.shape == (ch, h, w)
    assert np.array_equal(act, exp)


def test_vardct_golden_issue_24_all_keyframes(oracle):
    """The reference's only VarDCT fixture whose golden buffer is in the tree (SURVEY section 8c (4)): a 1 x 1 grayscale
    VarDCT animation, nine keyframes, replayed like tests/decode/mod.rs:29-86 (per keyframe: marker 0, then the planes
    as u16 = (v * 65535 + 0.5)). The reference allows 0.004 * 65535 = 262 for VarDCT; the oracle reproduces every
    sample exactly."""
    gold = oracle.zstd_decompress(fixture_bytes("issue_24", "output.buf.zst"))
    w, h, ch = struct.unpack("<III", gold[:12])
    img = oracle.OracleImage(fixture_bytes("issue_24", "input.jxl"))
    assert (w, h, ch) == (1, 1, 1) and img.num_frames == 9
    off = 12
    for i in range(img.num_frames):
        assert gold[off] == 0
        planes, _, is_vardct = img.frame(i)
        assert is_vardct and planes.shape == (ch, h, w)
        exp = np.frombuffer(gold, dtype="<u2", count=w * h * ch, offset=off + 1).reshape(ch, h, w)
        act = (planes * np.float32(65535.0) + np.float32(0.5)).astype(np.uint16)
        assert np.array_equal(act, exp), f"keyframe {i}"
        off += 1 + w * h * ch * 2
    assert gold[off] == 0xFF and off + 1 == len(gold)


def test_vardct_conformance_opsin_inverse(oracle):
    """ISO 18181-3 level of agreement with libjxl's reference rendering (8-bit ref.png):
    crates/jxl-oxide-tests/tests/conformance/mod.rs:139-368 uses peak 0.004 for VarDCT."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("opsin_inverse", "input.jxl"), threads=4)
    planes, ncol, is_vardct = img.frame(0)
    assert is_vardct and ncol == 3
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("opsin_inverse", "ref.png")))).astype(np.float32) / 255.0
    ref = np.moveaxis(ref, 2, 0)
    diff = np.abs(np.clip(planes, 0.0, 1.0) - ref)
    assert diff.max() <= 0.004
    assert math.sqrt(float((diff ** 2).mean())) <= 0.004


def test_vardct_conformance_upsampling(oracle):
    """2x non-separable upsampling (features/upsampling.rs) + alpha, against libjxl's 8-bit rendering."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("upsampling", "input.jxl"), threads=4)
    planes, ncol, is_vardct = img.frame(0)
    assert is_vardct and planes.shape == (4, 600, 800)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("upsampling", "ref.png")))).astype(np.float32) / 255.0
    ref = np.moveaxis(ref, 2, 0)
    diff = np.abs(np.clip(planes, 0.0, 1.0) - ref)
    assert diff.max() <= 0.004
    assert math.sqrt(float((diff ** 2).mean())) <= 0.004


def test_vardct_conformance_noise(oracle):
    """Noise synthesis (features/noise.rs): XorShift128+ field per group, 5x5 high-pass, strength LUT. The
    field is deterministic, so libjxl's rendering pins the generator, its seeds and the placement."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("noise", "input.jxl"), threads=4)
    planes, ncol, is_vardct = img.frame(0)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("noise", "ref.png")))).astype(np.float32) / 255.0
    ref = np.moveaxis(ref, 2, 0)
    diff = np.abs(np.clip(planes, 0.0, 1.0) - ref)
    assert diff.max() <= 0.004
    assert math.sqrt(float((diff ** 2).mean())) <= 0.004


def test_patches_lossless_exact(oracle):
    """Reference-only frames + patch dictionary (jxl-frame/src/data/patch.rs, jxl-render/src/blend.rs:418-606)
    on a lossless image: every 8-bit sample of libjxl's rendering is reproduced."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("patches_lossless", "input.jxl"), threads=4)
    planes, ncol, _ = img.frame(0)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("patches_lossless", "ref.png"))))
    ref = np.moveaxis(ref, 2, 0)
    act = np.rint(np.clip(planes[:ref.shape[0]], 0, 1) * 255.0).astype(np.uint8)
    assert np.array_equal(act, ref)


def test_vardct_conformance_bike(oracle):
    """The conformance suite's photograph: VarDCT + patches from a reference frame + BT.709 output
    transfer (jxl-color/src/tf/bt709.rs). Compared on a crop of libjxl's 8-bit rendering (peak limit 0.007)."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("bike", "input.jxl"), threads=8)
    planes, ncol, is_vardct = img.frame(0)
    assert is_vardct and planes.shape == (3, 2560, 2048)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("bike", "ref_crop_700_900.png")))).astype(np.float32) / 255.0
    ref = np.moveaxis(ref, 2, 0)
    diff = np.abs(np.clip(planes[:, 900:1540, 700:1340], 0.0, 1.0) - ref)
    assert diff.max() <= 0.007
    assert math.sqrt(float((diff ** 2).mean())) <= 0.002


def test_layers_blending_and_orientation_sunset_logo(oracle):
    """Cropped layers composed onto the canvas (jxl-render/src/blend.rs) and orientation 7 through
    ImageStream::write_to_buffer (fb.rs:387-401): libjxl's rendering is reproduced at 8 bits."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("sunset_logo", "input.jxl"), threads=4)
    assert img.orientation == 7
    buf = img.frame_to_buffer(0, np.uint16, 0).astype(np.float32) / 65535.0
    assert buf.shape == (1386, 924, 4)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("sunset_logo", "ref_crop_200_400.png")))).astype(np.float32) / 255.0
    assert np.abs(buf[400:912, 200:712] - ref).max() <= 0.004


def test_animation_frames_icos4d(oracle):
    """48 cropped frames blended over reference slots; three of them against the reference APNG."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("animation_icos4d", "input.jxl"), threads=4)
    assert img.num_frames == 48
    for k in (0, 17, 47):
        ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("animation_icos4d", "ref_frame_%02d.png" % k)))).astype(np.float32) / 255.0
        got = np.moveaxis(np.clip(img.frame(k)[0], 0.0, 1.0), 0, 2)
        assert np.abs(got - ref).max() <= 0.004, k


def test_jpeg_transcode_ycbcr_444(oracle):
    """JPEG-transcoded frame: raw (Modular-coded) dequant tables (dequant.rs:367-381, 537-559), YCbCr -> RGB
    (jxl-color/src/ycbcr.rs) and orientation 5, against libjxl's rendering."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("bench_oriented_brg", "input.jxl"), threads=4)
    assert img.orientation == 5
    buf = img.frame_to_buffer(0, np.float32, 0)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("bench_oriented_brg", "ref.png")))).astype(np.float32) / 255.0
    assert buf.shape == ref.shape == (500, 606, 3)
    assert np.abs(np.clip(buf, 0.0, 1.0) - ref).max() <= 0.004
    gray = oracle.OracleImage(fixture_bytes("grayscale_jpeg", "input.jxl"), threads=4)
    planes, ncol, _ = gray.frame(0)
    assert planes.shape == (1, 200, 200) and ncol == 1


def test_jpeg_transcode_ycbcr_420(oracle):
    """4:2:0 JPEG transcode: per-channel block grids (ChannelShift::from_jpeg_upsampling), shifted HF decode /
    dequant / IDCT, the 0.75 / 0.25 chroma upsampling (filter/ycbcr.rs) and YCbCr -> RGB, against libjxl's rendering
    (an interior crop and the bottom-right corner, where the edge replication shows)."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("cafe", "input.jxl"), threads=8)
    planes, ncol, _ = img.frame(0)
    assert planes.shape == (3, 1600, 1280)
    got = np.moveaxis(np.clip(planes, 0.0, 1.0), 0, 2)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("cafe", "ref_crop_600_800.png")))).astype(np.float32) / 255.0
    assert np.abs(got[800:1312, 600:1112] - ref).max() <= 0.004
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("cafe", "ref_crop_corner.png")))).astype(np.float32) / 255.0
    assert np.abs(got[1344:1600, 1024:1280] - ref).max() <= 0.004


def test_spot_colours_in_the_image_stream(oracle):
    """16-bit RGB + alpha + two spot-colour channels: ImageStream mixes the spots into RGB while writing
    (fb.rs:246-283, 335-362) and appends the alpha channel; planar access leaves all six channels untouched."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("spot", "input.jxl"), threads=4)
    assert img.frame(0)[0].shape == (6, 400, 600)
    buf = np.clip(img.frame_to_buffer(0, np.float32, 0), 0.0, 1.0)
    assert buf.shape == (400, 600, 4)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("spot", "ref_crop_150_50.png")))).astype(np.float32) / 255.0
    assert np.abs(buf[50:350, 150:450] - ref).max() <= 0.004


def test_delta_palette_exact(oracle):
    """Lossy palette: a palette without explicit colours, implicit and delta entries, and the serial prediction pass
    over the samples below nb_deltas (transform/palette.rs:26-152) - libjxl's 8-bit rendering is reproduced exactly."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("delta_palette", "input.jxl"), threads=4)
    planes, ncol, _ = img.frame(0)
    assert planes.shape == (3, 751, 555)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("delta_palette", "ref_crop_100_200.png")))).astype(np.int32)
    got = np.rint(np.clip(np.moveaxis(planes, 0, 2)[200:500, 100:400], 0.0, 1.0) * 255.0).astype(np.int32)
    assert np.array_equal(got, ref)


# sha256 of the embedded profile ("original.icc" in the conformance suite's test.json files)
ICC_SHA256 = {
    "bench_oriented_brg": "6603ae12a4ac",
    "cafe": "bef95ce5cdb1",
    "grayscale": "3f62598dfd40",
    "grayscale_jpeg": "78001f4bf342",
    "patches_lossless": "3a10bcd8e4c3",
    "spot": "ce0caee95061",
    "cmyk_layers": "4855b8fabb96",
    "patches": "3a10bcd8e4c3",
    "progressive": "bef95ce5cdb1",
}


@pytest.mark.parametrize("name", sorted(ICC_SHA256))
def test_embedded_icc_profiles_are_reconstructed_exactly(oracle, name):
    """ICC stream decode (jxl-color/src/icc/decode.rs): header prediction, tag-list commands, shuffles and Nth-order
    predictors - the reconstructed profiles hash to the conformance suite's `original.icc` digests."""
    import hashlib
    icc = oracle.OracleImage(fixture_bytes(name, "input.jxl"), threads=2).original_icc()
    assert len(icc) >= 128 and icc[36:40] == b"acsp"
    assert hashlib.sha256(icc).hexdigest().startswith(ICC_SHA256[name])


def test_pq_inverse_eotf_known_answers(oracle):
    """The reference's pq_inverse_eotf_100k_generic (jxl-color/src/tf/pq.rs:460-478): 100 000 linear values at a
    10 000-nit intensity target against the closed-form ST 2084 curve, |diff| < 1e-6."""
    import ctypes
    L = oracle.lib()
    v = (np.arange(100000, dtype=np.float32) * np.float32(1e-5)).astype(np.float32)
    lin = v.astype(np.float64)
    L.jxlo_linear_to_pq.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float]
    L.jxlo_linear_to_pq(v.ctypes.data, v.size, 10000.0)
    m1, m2, c1, c2, c3 = 2610 / 16384, 2523 / 4096 * 128, 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32
    want = ((c1 + c2 * lin ** m1) / (1 + c3 * lin ** m1)) ** m2
    assert np.abs(v - want).max() < 1e-6


def test_icc_recognition_known_answers(oracle):
    """The reference's own unit tests for parse_icc (crates/jxl-color/src/icc/parse.rs:566-671) on its test profiles:
    colour space, white point, primaries, transfer function and rendering intent of each."""
    RGB, GREY, D65, SRGB_PRIM, CUSTOM = 0, 1, 1, 1, 2
    TF_GAMMA, TF_709, TF_LINEAR, TF_SRGB = 0, 1, 8, 13
    PERCEPTUAL, RELATIVE = 0, 1
    cases = {
        "srgb-rel.icc": (RGB, D65, SRGB_PRIM, TF_SRGB, RELATIVE),
        "srgb-bt709-per.icc": (RGB, D65, SRGB_PRIM, TF_709, PERCEPTUAL),
        "srgb-gamma22-rel.icc": (RGB, D65, SRGB_PRIM, TF_GAMMA, RELATIVE),
        "srgb-linear-rel.icc": (RGB, D65, SRGB_PRIM, TF_LINEAR, RELATIVE),
        "gray-d65-srgb-rel.icc": (GREY, D65, None, TF_SRGB, RELATIVE),
        "gray-d65-linear-rel.icc": (GREY, D65, None, TF_LINEAR, RELATIVE),
    }
    for name, (cs, wp, prim, tf, intent) in cases.items():
        st, e = oracle.icc_to_enum(fixture_bytes("icc", name))
        assert st == 0, name
        assert (e["colour_space"], e["white_point"], e["tf"], e["rendering_intent"]) == (cs, wp, tf, intent), (name, e)
        if prim is not None:
            assert e["primaries"] == prim, (name, e)
        if tf == TF_GAMMA:  # 0x23332 / 65536 = 2.19998...: Gamma { g in 21999000..=22001000, inverted: false }
            assert 21999000 <= e["gamma"] <= 22001000 and e["gamma_inverted"] == 0
    # ProPhoto (ROMM) primaries, D50 white, gamma 1.8: custom xy values, still an enum encoding
    st, e = oracle.icc_to_enum(fixture_bytes("icc", "prophoto-gamma18-rel.icc"))
    assert st == 0 and e["colour_space"] == RGB and e["primaries"] == CUSTOM and e["white_point"] == CUSTOM
    assert e["tf"] == TF_GAMMA and 17990000 <= e["gamma"] <= 18010000
    # truncated / foreign data is malformed, not a crash
    assert oracle.icc_to_enum(b"\0" * 64)[0] == 2
    assert oracle.icc_to_enum(fixture_bytes("icc", "srgb-rel.icc")[:200])[0] == 2


def test_xyb_grayscale_with_icc_profile(oracle):
    """XYB image tagged with a gray ICC profile whose curve is tabulated: no enum encoding describes it, so the
    render target is gray sRGB (jxl-render/src/lib.rs:104-150) - gamut map, D65 luma row, sRGB curve, one channel."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("grayscale", "input.jxl"), threads=4)
    planes, ncol, _ = img.frame(0)
    assert planes.shape == (1, 200, 200) and ncol == 1
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("grayscale", "ref.png")))).astype(np.float32) / 255.0
    assert np.abs(np.clip(planes[0], 0.0, 1.0) - ref).max() <= 0.004


def test_lossless_float_samples_exact(oracle):
    """32-bit float Modular image (jxl-image/src/lib.rs:464-488 sample reinterpretation): every sample equals the
    conformance suite's ref.pfm bit for bit (values span -2 .. 1.99)."""
    import hashlib
    planes = oracle.OracleImage(fixture_bytes("lossless_pfm", "input.jxl"), threads=4).frame(0)[0]
    assert planes.shape == (3, 500, 500)
    digest = hashlib.sha256(np.ascontiguousarray(np.moveaxis(planes, 0, 2), dtype="<f4").tobytes()).hexdigest()
    assert digest == fixture_bytes("lossless_pfm", "ref_f32_sha256.txt").decode().strip()


def test_alpha_images_against_libjxl_renderings(oracle):
    """Straight and premultiplied alpha (ExtraChannelInfo::alpha_associated), 8 and 16 bit, Modular and VarDCT."""
    from PIL import Image
    import io

    def png(*parts):
        return np.asarray(Image.open(io.BytesIO(fixture_bytes(*parts)))).astype(np.float32) / 255.0

    for name in ("alpha_triangles", "alpha_nonpremultiplied"):
        buf = np.clip(oracle.OracleImage(fixture_bytes(name, "input.jxl"), threads=4).frame_to_buffer(0, np.float32, 0), 0, 1)
        assert np.abs(buf - png(name, "ref.png")).max() <= 0.004, name
    # the PNG holds straight alpha, the decoder (like jxl-oxide) leaves the colours premultiplied
    buf = oracle.OracleImage(fixture_bytes("alpha_premultiplied", "input.jxl"), threads=4).frame_to_buffer(0, np.float32, 0)[256:768, 256:768]
    ref = png("alpha_premultiplied", "ref_crop_256_256.png")
    assert np.abs(buf[..., 3] - ref[..., 3]).max() <= 0.004
    opaque = buf[..., 3] > 0.05
    straight = np.clip(buf[..., :3] / np.maximum(buf[..., 3:4], 1e-6), 0, 1)
    assert np.abs(straight - ref[..., :3])[opaque].max() <= 0.004
    buf = np.clip(oracle.OracleImage(fixture_bytes("bicycles", "input.jxl"), threads=4).frame_to_buffer(0, np.float32, 0), 0, 1)
    assert np.abs(buf[100:612, 300:812] - png("bicycles", "ref_crop_300_100.png")).max() <= 0.004


def test_palette_animation_newtons_cradle(oracle):
    """36-frame Modular animation transcoded from a GIF (palette + blending over the previous canvas): the first frame
    equals the GIF's exactly; a later one everywhere except the handful of pixels where PIL composes transparent GIF
    pixels differently."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("animation_newtons_cradle", "input.jxl"), threads=4)
    assert img.num_frames == 36
    for k, tol in ((0, 0.0), (10, 0.01)):
        ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("animation_newtons_cradle", "ref_frame_%02d.png" % k)))).astype(np.float32) / 255.0
        got = np.moveaxis(np.clip(img.frame(k)[0], 0, 1), 0, 2)
        assert (np.abs(got - ref).max(axis=2) > 0.004).mean() <= tol, k


def test_jpeg_transcode_odd_block_count(oracle):
    """228 x 256 4:2:0 transcode (the reference's issue_425): 28.5 luma blocks per row, so the block grid is rounded
    up to an even count (hf_metadata.rs:70-80) and the chroma edge sample is replicated. The source JPEG decoded by
    libjpeg agrees to within the two decoders' IDCT / upsampling differences."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("issue_425", "input.jxl"), threads=4)
    buf = np.clip(img.frame_to_buffer(0, np.float32, 0), 0, 1)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("issue_425", "ref.jpg"))).convert("RGB")).astype(np.float32) / 255.0
    assert buf.shape == ref.shape == (256, 228, 3)
    assert np.abs(buf - ref).max() <= 0.02 and np.sqrt(((buf - ref) ** 2).mean()) <= 0.004


def test_cmyk_image_stream_carries_the_black_channel(oracle):
    """CMYK image (the ICC profile's data colour space says so): ImageStream = C, M, Y, then K, then alpha
    (fb.rs:205-243). No CMS here, so the samples stay CMYK."""
    img = oracle.OracleImage(fixture_bytes("cmyk_layers", "input.jxl"), threads=4)
    assert img.frame(0)[0].shape == (5, 512, 512)
    assert img.frame_to_buffer(0, np.uint8, 0).shape == (512, 512, 5)


def test_icc_tagged_xyb_images_fall_back_to_srgb(oracle):
    """XYB images whose ICC profile no enum encoding describes (`chrm` tag, tabulated curves) render to sRGB, as
    jxl-oxide does without a CMS (jxl-render/src/lib.rs:104-150); the large Squeeze-progressive Modular frame and
    the VarDCT frame with patches and alpha decode to finite, in-range pixels."""
    for name, shape in (("progressive", (3, 2704, 4064)), ("patches", (4, 1096, 1600))):
        planes = oracle.OracleImage(fixture_bytes(name, "input.jxl"), threads=8).frame(0)[0]
        assert planes.shape == shape and np.isfinite(planes).all()
        assert -0.5 < float(planes.min()) and float(planes.max()) < 1.5  # wide-gamut content leaves sRGB's [0, 1]


def test_animation_splines(oracle):
    """60 frames whose only content is splines drawn over a flat background (features/spline.rs): quantised control
    points, Catmull-Rom upsampling, unit arc sampling and the erf splat, against three frames of the reference APNG."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("animation_spline", "input.jxl"), threads=4)
    assert img.num_frames == 60
    for k in (0, 23, 59):
        ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("animation_spline", "ref_frame_%02d.png" % k)))).astype(np.float32) / 255.0
        got = np.moveaxis(np.clip(img.frame(k)[0], 0.0, 1.0), 0, 2)
        assert np.abs(got - ref).max() <= 0.004, k


def test_blend_modes_alpha_plane(oracle):
    """Replace / Blend / Add / Mul / MulAdd layers (blend.rs:55-103, 550-727). The alpha plane of libjxl's
    rendering is reproduced everywhere; the colour planes wherever the last layer's weight stayed in [0, 1]
    (the reference decoder does not clamp it when the frame's clamp flag is off, the PNG's producer did)."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("blendmodes", "input.jxl"), threads=4)
    planes, _, _ = img.frame(0)
    ref = np.moveaxis(np.asarray(Image.open(io.BytesIO(fixture_bytes("blendmodes", "ref.png")))).astype(np.float32) / 255.0, 2, 0)
    diff = np.abs(np.clip(planes, 0.0, 1.0) - ref)
    assert diff[3].max() <= 0.004
    assert float((diff[:3].max(axis=0) <= 0.004).mean()) > 0.25


def test_grayscale_modular_with_filters(oracle):
    """One-channel Modular frame (Squeeze) whose restoration filters run on a cloned gray triple
    (jxl-render/src/render.rs:74-134)."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("grayscale_public_university", "input.jxl"), threads=8)
    planes, ncol, _ = img.frame(0)
    assert planes.shape == (1, 1620, 2880)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("grayscale_public_university", "ref_crop_1000_500.png")))).astype(np.float32) / 255.0
    assert np.abs(np.clip(planes[0, 500:1012, 1000:1512], 0.0, 1.0) - ref).max() <= 0.004


def test_lz77_modular_vs_png(oracle):
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("lz77_flower", "input.jxl"))
    planes, ncol, _ = img.frame(0)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("lz77_flower", "ref.png"))))
    ref = np.moveaxis(ref, 2, 0)[:ncol]
    act = np.rint(planes[:ncol] * 255.0).astype(np.uint8)
    assert np.array_equal(act, ref)


def _dct2_f64(x):
    n = len(x)
    out = []
    for k in range(n):
        s = sum(x[i] * math.cos(math.pi * (i + 0.5) * k / n) for i in range(n))
        scale = (1.0 / n) if k == 0 else (math.sqrt(2.0) / n)
        out.append(s * scale)
    return out


def _dct3_f64(c):
    n = len(c)
    return [c[0] + sum(math.sqrt(2.0) * c[k] * math.cos(math.pi * (i + 0.5) * k / n) for k in range(1, n)) for i in range(n)]


@pytest.mark.parametrize("n", [2, 4, 8, 16, 32])
@pytest.mark.parametrize("forward", [True, False])
def test_dct_known_answers(oracle, n, forward):
    """Same criterion as the reference's unit tests (generic/dct.rs:295-436): compare against the
    f64 closed form after quantising to 2^-16."""
    L = oracle.lib()
    L.jxlo_dct_2d.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
    rng = np.random.default_rng(n * 2 + int(forward))
    x = rng.uniform(-1.0, 1.0, size=n).astype(np.float32)
    buf = x.copy()
    L.jxlo_dct_2d(buf.ctypes.data, n, 1, int(forward))
    exp = _dct2_f64([float(v) for v in x]) if forward else _dct3_f64([float(v) for v in x])
    got = (buf.astype(np.float64) * 65536).astype(np.int64)
    want = (np.array(exp) * 65536).astype(np.int64)
    assert np.abs(got - want).max() <= 1


@pytest.mark.parametrize("n", [64, 128, 256])
@pytest.mark.parametrize("forward", [True, False])
def test_dct_known_answers_large(oracle, n, forward):
    """The 64-, 128- and 256-point transforms of DCT64 .. DCT256 against the f64 closed form, on dense uniform +-1 inputs
    as in the 2^-16 test above. That criterion does not hold here (the 256-point inverse is up to ~17 such units off), so
    the bound is float32 roundoff: the recursion has log2(n) butterfly levels, each rounding an add and a multiply by a
    constant, and a level's rounding error is scaled by its secant factor 1 / (2 cos(.)) before it reaches the output.
    Allowed: 8 units of 2^-24 per level, relative to the l1 norm of the terms an output sums (sum_k alpha_k |c_k| for the
    inverse, sqrt(2) / n sum_i |x_i| for the forward transform); the measured worst case is under half of that."""
    L = oracle.lib()
    L.jxlo_dct_2d.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
    m = np.cos(np.pi * (np.arange(n)[:, None] + 0.5) * np.arange(n)[None, :] / n)  # m[i, k]: sample i of basis k
    alpha = np.r_[1.0, np.full(n - 1, math.sqrt(2.0))]
    rng = np.random.default_rng(n * 2 + int(forward))
    for _ in range(16):
        x = rng.uniform(-1.0, 1.0, size=n).astype(np.float32)
        buf = x.copy()
        L.jxlo_dct_2d(buf.ctypes.data, n, 1, int(forward))
        x64 = x.astype(np.float64)
        if forward:
            want, l1 = (m.T @ x64) * alpha / n, math.sqrt(2.0) / n * np.abs(x64).sum()
        else:
            want, l1 = m @ (alpha * x64), (alpha * np.abs(x64)).sum()
        bound = 8 * math.log2(n) * 2.0 ** -24 * l1
        assert np.abs(buf.astype(np.float64) - want).max() <= bound


def test_threads_do_not_change_results(oracle):
    data = fixture_bytes("opsin_inverse", "input.jxl")
    a, _, _ = oracle.OracleImage(data, threads=1).frame(0)
    b, _, _ = oracle.OracleImage(data, threads=4).frame(0)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_truncated_and_garbage_inputs_error_cleanly(oracle):
    """Decode errors are values, never crashes (reference: fuzz_findings tests)."""
    data = fixture_bytes("squeeze_edge", "input.jxl")
    for cut in (2, 10, len(data) // 2):
        with pytest.raises(oracle.OracleError):
            oracle.OracleImage(data[:cut])
    with pytest.raises(oracle.OracleError):
        oracle.OracleImage(b"\x00" * 64)


def test_synthetic_encoder_roundtrips_through_oracle(oracle):
    """tools/synth_enc.cc writes a stream whose ANS final states, TOC and block layout the decoder
    accepts; the generator is deterministic per seed."""
    import bench
    a = bench.synth_frame(520, 392, 11)
    b = bench.synth_frame(520, 392, 11)
    assert a == b
    img = oracle.OracleImage(a, threads=4)
    planes, ncol, is_vardct = img.frame(0)
    assert is_vardct and planes.shape == (3, 392, 520) and np.isfinite(planes).all()


def test_progressive_passes_sum_to_the_single_pass_image(oracle):
    """The same coefficients sent in one, two or three passes (shifts 0 / 1,0 / 2,1,0; hf_coeff.rs:246 `<< coeff_shift`,
    per-pass histograms and non-zero contexts) decode to bit-identical pixels."""
    import bench
    one = oracle.OracleImage(bench.synth_frame(600, 500, 5), threads=4).frame(0)[0]
    for passes in ("2", "3"):
        data = bench.synth_frame(600, 500, 5, extra=("--passes", passes))
        got = oracle.OracleImage(data, threads=4).frame(0)[0]
        assert np.array_equal(got.view(np.uint32), one.view(np.uint32)), passes


def test_enum_colour_targets_against_float64_colour_math(oracle):
    """XYB -> P3 / BT.2100 / custom primaries, DCI / custom white points, Grey, gamma and DCI transfer functions
    (jxl-color/src/convert.rs:397-466, ciexyz.rs, gamut.rs, tf.rs). No reference rendering with such an enum encoding
    exists offline, so the check is numerical: the decoder's linear-sRGB output pushed through textbook float64
    colour math (chromaticity matrices, Bradford adaptation, analytic transfer curves) must agree."""
    import bench
    D65 = (0.3127, 0.329)
    SRGB = ((0.639998686, 0.330010138), (0.300003784, 0.600003357), (0.150002046, 0.059997204))
    P3 = ((0.680, 0.320), (0.265, 0.690), (0.150, 0.060))
    BT2100 = ((0.708, 0.292), (0.170, 0.797), (0.131, 0.046))

    def wxyz(w):
        return np.array([w[0] / w[1], 1.0, (1 - w[0] - w[1]) / w[1]])

    def rgb2xyz(prim, wp):
        m = np.array([[q[0] for q in prim], [q[1] for q in prim], [1 - q[0] - q[1] for q in prim]])
        return m * np.linalg.solve(m, wxyz(wp))[None, :]

    br = np.array([[0.8951, 0.2664, -0.1614], [-0.7502, 1.7135, 0.0367], [0.0389, -0.0685, 1.0296]])

    def adapt(f, t):
        return np.linalg.inv(br) @ np.diag((br @ wxyz(t)) / (br @ wxyz(f))) @ br

    def gamut(rgb, lum, sat=0.3):  # gamut.rs:4-46
        y = (rgb * lum[:, None, None]).sum(0)
        gs, gl = np.zeros_like(y), np.zeros_like(y)
        for v in rgb:
            d = v - y
            inv = 1.0 / np.where(d == 0, 1.0, d)
            vo = v * inv
            gs = np.where(d >= 0, gs, np.maximum(gs, vo))
            gl = np.maximum(np.where(d <= 0, gs, vo - inv), gl)
        mix = np.clip(sat * (gs - gl) + gl, 0, 1)
        return (mix * (y - rgb) + rgb) / np.maximum(1.0, rgb.max(0))

    def srgb_oetf(v):
        a = np.abs(v)
        return np.sign(v) * np.where(a <= 0.0031308, 12.92 * a, 1.055 * np.power(a, 1 / 2.4) - 0.055)

    def gam(v, g):
        return np.where(v <= 1e-7, 0.0, np.power(np.maximum(v, 1e-30), g))

    lin = oracle.OracleImage(bench.synth_frame(600, 500, 5), output_colour=1, threads=4).frame(0)[0].astype(np.float64)
    to_xyz = rgb2xyz(SRGB, D65)
    g = gamut(lin, to_xyz[1])
    cases = {"p3": (P3, D65, srgb_oetf, 2e-4), "rec2020-gamma": (BT2100, D65, lambda v: gam(v, 0.4166667), 5e-6),
             "dci": (P3, (0.314, 0.351), lambda v: gam(v, 1 / 2.6), 5e-6),
             "custom": (((0.64, 0.33), (0.21, 0.71), (0.15, 0.06)), (0.3457, 0.3585), lambda v: gam(v, 0.4545455), 5e-6)}
    for name, (prim, wp, tf, tol) in cases.items():
        m = np.linalg.inv(rgb2xyz(prim, wp)) @ adapt(D65, wp) @ to_xyz
        want = tf(np.einsum("ij,jhw->ihw", m, g))
        got = oracle.OracleImage(bench.synth_frame(600, 500, 5, extra=("--colour", name)), threads=4).frame(0)[0]
        assert got.shape == want.shape and np.abs(got - want).max() <= tol, name
    # PQ (SMPTE ST 2084 inverse EOTF) on BT.2100 primaries, 1000-nit intensity target: an HDR target, no tone mapping
    data = bench.synth_frame(600, 500, 5, extra=("--colour", "pq"))
    hdr = oracle.OracleImage(data, output_colour=1, threads=4).frame(0)[0].astype(np.float64)
    v = np.einsum("ij,jhw->ihw", np.linalg.inv(rgb2xyz(BT2100, D65)) @ to_xyz, gamut(hdr, to_xyz[1]))
    y = np.abs(v) * 1000.0 / 10000.0
    m1, m2, c1, c2, c3 = 2610 / 16384, 2523 / 4096 * 128, 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32
    want = np.sign(v) * ((c1 + c2 * y ** m1) / (1 + c3 * y ** m1)) ** m2
    assert np.abs(oracle.OracleImage(data, threads=4).frame(0)[0] - want).max() <= 2e-6
    got = oracle.OracleImage(bench.synth_frame(600, 500, 5, extra=("--colour", "gray")), threads=4).frame(0)[0]
    assert got.shape == (1, 500, 600)
    assert np.abs(got[0] - srgb_oetf(np.einsum("ij,jhw->ihw", to_xyz, g))[1]).max() <= 2e-4


def _fuzz_files():
    import glob
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fuzz_findings")
    return sorted(glob.glob(os.path.join(here, "*.fuzz")))


def test_fuzz_findings_are_clean_errors(oracle):
    """The reference's fuzz corpus (tests/fuzz_findings): every input ends in a decode or an error
    VALUE with a known code - never a crash, a hang or an unclassified exception."""
    files = _fuzz_files()
    assert len(files) >= 60
    for f in files:
        data = open(f, "rb").read()
        try:
            oracle.OracleImage(data, threads=2).close()
        except oracle.OracleError as e:
            assert e.code in (1, 2, 3), (f, str(e))


def test_write_to_buffer_u8_matches_png(oracle):
    """ImageStream::write_to_buffer::<u8> (fb.rs:309-410) of a lossless 8-bit image reproduces the PNG bytes."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("lz77_flower", "input.jxl"))
    buf = img.frame_to_buffer(0, np.uint8, 1)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("lz77_flower", "ref.png"))))
    assert buf.shape[:2] == ref.shape[:2]
    assert np.array_equal(buf[:, :, :ref.shape[2]], ref[:, :, :buf.shape[2]])
    rot = img.frame_to_buffer(0, np.uint8, 6)  # orientation 6: (x, y) <- (y, w - x - 1)
    assert rot.shape[0] == buf.shape[1] and rot.shape[1] == buf.shape[0]
    assert np.array_equal(rot, np.rot90(buf, k=-1)) or np.array_equal(rot, np.rot90(buf, k=1))


def test_lf_frame_streams_decode(oracle):
    """A frame that takes its LF image from a preceding Modular LF frame (use_lf_frame,
    jxl-render/src/lib.rs:294-318, vardct/mod.rs:175-180): two frames in the codestream, one shown."""
    import bench
    data = bench.synth_frame(1000, 600, 7, extra=("--lf-frame",))
    img = oracle.OracleImage(data, threads=4, output_colour=2)
    assert img.num_frames == 1
    planes, ncol, is_vardct = img.frame(0)
    assert is_vardct and planes.shape == (3, 600, 1000) and np.isfinite(planes).all()
    assert 0.2 < float(planes[1].max()) < 1.0  # luma comes from the LF frame's samples


def test_epf_iteration_counts_change_the_image(oracle):
    """tools/synth_enc.cc --epf-iters 0 / 1 / 3 (explicit restoration filter) next to the all-default filter (2): each
    count decodes to a different image, ordered by how much smoothing it applies."""
    import bench
    imgs = {}
    for it in (0, 1, 2, 3):
        extra = () if it == 2 else ("--epf-iters", str(it))
        imgs[it] = oracle.OracleImage(bench.synth_frame(520, 392, 11, extra=extra), threads=4).frame(0)[0]
    for a in range(4):
        for b in range(a + 1, 4):
            assert not np.array_equal(imgs[a], imgs[b])
    # more smoothing iterations move the image further from the unfiltered one
    d = [float(np.abs(imgs[it] - imgs[0]).mean()) for it in (1, 2, 3)]
    assert 0 < d[0] < d[1] < d[2]


@pytest.mark.parametrize("presets", [2, 5])
def test_hf_presets_select_their_own_cluster_maps(oracle, presets):
    """No fixture of the reference uses more than one HF preset (hf_pass.rs / hf_coeff.rs:60-75), so tools/synth_enc.cc
    --hf-presets N codes group g with preset g % N, every preset owning a differently clustered slice of the pass code:
    the coefficients are the same, so the image must equal the single-preset stream's bit for bit."""
    import bench
    one = oracle.OracleImage(bench.synth_frame(1000, 600, 7), threads=4).frame(0)[0]
    many = oracle.OracleImage(bench.synth_frame(1000, 600, 7, extra=("--hf-presets", str(presets))), threads=4).frame(0)[0]
    assert np.array_equal(one.view(np.uint32), many.view(np.uint32))


def test_jpeg_transcode_420_full_size(oracle):
    """The reference's genshin_ycbcr_420 (2560 x 1440, 60 groups, chroma at half resolution both ways; its golden buffer
    is not in the tree): a 256 x 256 crop of the source JPEG as libjpeg decodes it agrees to within the two decoders'
    IDCT / upsampling differences, as for issue_425."""
    from PIL import Image
    import io
    img = oracle.OracleImage(fixture_bytes("genshin_ycbcr_420", "input.jxl"), threads=4)
    buf = np.clip(img.frame_to_buffer(0, np.float32, 0), 0, 1)
    assert buf.shape == (1440, 2560, 3)
    ref = np.asarray(Image.open(io.BytesIO(fixture_bytes("genshin_ycbcr_420", "refjpg_crop_1000_600.png")))).astype(np.float32) / 255.0
    crop = buf[600:856, 1000:1256]
    assert np.abs(crop - ref).max() <= 0.03 and np.sqrt(((crop - ref) ** 2).mean()) <= 0.004
