"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same inputs.

Bar (BASELINE.json north_star): bit-exact for the integer/Modular path, <= 1 ULP for the VarDCT
float pipeline. The kernels reproduce the reference's float op order, so VarDCT is asserted
bit-exact too (0 ULP), stage by stage.
"""
import numpy as np
import pytest

from conftest import fixture_bytes

pytestmark = pytest.mark.gpu

MODULAR = ["grayalpha", "squeeze_edge", "issue_311", "alpha_triangles", "bicycles", "lz77_flower", "patches_lossless", "sunset_logo", "blendmodes", "grayscale_public_university", "spot", "delta_palette", "lossless_pfm", "cmyk_layers", "progressive"]
MODULAR_BENCH = ["srgb.d0-e1.jxl", "minecraft.d0-e6.jxl"]
VARDCT = ["opsin_inverse", "alpha_premultiplied", "minecraft_vardct_e7", "upsampling", "noise", "bike", "bench_oriented_brg", "grayscale_jpeg", "cafe", "grayscale", "issue_425", "patches"]
VARDCT_BENCH = ["starrail.d1-e6.jxl", "nahida-motion.d1-e7.jxl"]
STAGES_F32 = ["lf", "hf_dequant", "idct", "jpeg_upsampled", "pre_filter", "gaborish", "epf", "upsampled", "patches", "splines", "noise", "rgb"]


def ulp_diff(a, b):
    a = a.view(np.int32).astype(np.int64)
    b = b.view(np.int32).astype(np.int64)
    a = np.where(a < 0, np.int64(-2147483648) - a, a)
    b = np.where(b < 0, np.int64(-2147483648) - b, b)
    return np.abs(a - b)


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


def _decode_both(dec, oracle, data, capture=False, output_colour=0):
    dec.set_capture(capture)
    dec.decode(data, output_colour=output_colour)
    got = dec.frame_planar(0)
    img = oracle.OracleImage(data, output_colour=output_colour, threads=8, capture=capture)
    want, ncol, is_vardct = img.frame(0)
    return got, want, img


@pytest.mark.parametrize("name", MODULAR)
def test_modular_bit_exact(dec, oracle, name):
    got, want, _ = _decode_both(dec, oracle, fixture_bytes(name, "input.jxl"))
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("name", MODULAR_BENCH)
def test_modular_bench_files_bit_exact(dec, oracle, name):
    got, want, _ = _decode_both(dec, oracle, fixture_bytes("benchmark-data", name))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def _check_vardct(dec, oracle, data):
    # production path: Gaborish + EPF + colour fused into one kernel -> final pixels only
    dec.set_fuse_filters(True)
    got, want, img = _decode_both(dec, oracle, data)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "fused filter chain differs"
    # stage by stage
    dec.set_fuse_filters(False)
    try:
        _check_vardct_stages(dec, oracle, data)
    finally:
        dec.set_fuse_filters(True)


def _check_vardct_stages(dec, oracle, data):
    got, want, img = _decode_both(dec, oracle, data, capture=True)
    # integer stage: HF coefficients must be identical
    for g, w in zip(dec.stage("hf_coeff", np.int32), img.stage("hf_coeff", np.int32)):
        assert np.array_equal(g, w), "HF coefficient decode differs"
    for st in STAGES_F32:
        gs, ws = dec.stage(st), img.stage(st)
        assert len(gs) == len(ws), st
        for c, (g, w) in enumerate(zip(gs, ws)):
            d = ulp_diff(g, w)
            assert d.max() == 0, f"stage {st} channel {c}: max ULP diff {d.max()} at {np.unravel_index(d.argmax(), d.shape)}"
    assert got.shape == want.shape
    assert ulp_diff(got, want).max() <= 1  # north_star tolerance
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("name", VARDCT)
def test_vardct_stagewise_bit_exact(dec, oracle, name):
    _check_vardct(dec, oracle, fixture_bytes(name, "input.jxl"))


@pytest.mark.parametrize("name", VARDCT_BENCH)
def test_vardct_bench_files_bit_exact(dec, oracle, name):
    _check_vardct(dec, oracle, fixture_bytes("benchmark-data", name))


def test_errors_are_values(dec):
    import jxl_oxide_b200
    data = fixture_bytes("squeeze_edge", "input.jxl")
    for bad in (data[:10], data[: len(data) // 2], b"\x00" * 64):
        with pytest.raises(jxl_oxide_b200.JxlError):
            dec.decode(bad)
    dec.decode(data)  # the decoder stays usable after errors
    assert dec.frame_planar(0).shape == (4, 513, 513)


def test_stage_entry_points_match_pipeline(dec, oracle):
    """Stage-level C-ABI calls (the reference's impls:: seams) on torch device tensors."""
    import torch
    import jxl_oxide_b200
    data = fixture_bytes("opsin_inverse", "input.jxl")
    img = oracle.OracleImage(data, threads=8, capture=True)
    pre = img.stage("pre_filter")
    gab = img.stage("gaborish")
    planes = [torch.from_numpy(p.copy()).cuda() for p in pre]
    dec.gaborish(planes, [[0.115169525, 0.061248592]] * 3)
    dec.sync()
    for p, w in zip(planes, gab):
        assert np.array_equal(p.cpu().numpy().view(np.uint32), w.view(np.uint32))
    # inverse RCT type 6 (YCgCo) against numpy wrapping arithmetic
    rng = np.random.default_rng(7)
    a, b, c = [rng.integers(-2000, 2000, size=(37, 53), dtype=np.int32) for _ in range(3)]
    t = [torch.from_numpy(x.copy()).cuda() for x in (a, b, c)]
    dec.rct_inverse(t, 6)
    dec.sync()
    tmp = a - (c >> 1)
    e = c + tmp
    f = tmp - (b >> 1)
    d = f + b
    for got, want in zip(t, (d, e, f)):
        assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("size,seed,extra", [((1000, 600), 5, ()), ((1544, 1032), 6, ("--lf-gradient",)),
                                             ((1000, 600), 7, ("--lf-frame",)), ((1000, 600), 5, ("--passes", "3"))])
def test_synthetic_vardct_frames_bit_exact(dec, oracle, size, seed, extra):
    """Frames from tools/synth_enc.cc (the bench workload generator): all 27 transform families,
    WP- or gradient-coded LF, EPF 2 iterations; an LF frame; HF coefficients split over three passes
    (pass_group.rs:150-170: later passes add `value << shift` to the coefficients of earlier ones)."""
    import bench
    _check_vardct(dec, oracle, bench.synth_frame(size[0], size[1], seed, extra=extra))


@pytest.mark.parametrize("colour", ["p3", "rec2020-gamma", "gray", "dci", "custom", "pq"])
def test_enum_colour_targets_bit_exact(dec, oracle, colour):
    """Non-sRGB enum output encodings: gamut mapping, the merged target matrix, XyzToLuma and the gamma transfer
    function of xyb_to_rgb_kernel (convert.rs:397-466) against the oracle, stage by stage."""
    import bench
    _check_vardct(dec, oracle, bench.synth_frame(712, 520, 9, extra=("--colour", colour)))


@pytest.mark.parametrize("output_colour", [1, 2])
def test_fused_filters_other_output_encodings(dec, oracle, output_colour):
    """Linear-sRGB and XYB outputs go through the fused Gaborish+EPF(+colour) kernel as well."""
    dec.set_fuse_filters(True)
    for name in ("opsin_inverse",):
        got, want, _ = _decode_both(dec, oracle, fixture_bytes(name, "input.jxl"), output_colour=output_colour)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fuzz_findings_are_clean_errors_on_device(dec, oracle):
    """Malformed inputs: the CUDA path returns the same kind of result as the oracle (decode or an
    error value of the same class) and the decoder stays usable."""
    import glob
    import os
    import jxl_oxide_b200
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fuzz_findings")
    files = sorted(glob.glob(os.path.join(here, "*.fuzz")))
    assert len(files) >= 60
    for f in files:
        data = open(f, "rb").read()
        want = want_px = got_px = None
        try:
            img = oracle.OracleImage(data, threads=2)
            if img.num_frames:
                want_px = img.frame(0)[0]
            img.close()
        except oracle.OracleError as e:
            want = e.code
        got = None
        try:
            dec.decode(data)
            if dec.num_frames():
                got_px = dec.frame_planar(0)
            dec.release_frames()
        except jxl_oxide_b200.JxlError as e:
            got = e.code
        if want_px is not None and got_px is not None:  # both decode: the same pixels, bit for bit
            assert got_px.shape == want_px.shape, os.path.basename(f)
            assert np.array_equal(got_px.view(np.uint32), want_px.view(np.uint32)), os.path.basename(f)
        # device-side detection reports DEVICE_DECODE (6) where the host oracle says BITSTREAM (1)
        norm = {6: 1}
        assert norm.get(got, got) == norm.get(want, want), (os.path.basename(f), got, want)
    dec.decode(fixture_bytes("grayalpha", "input.jxl"))
    assert dec.frame_planar(0).shape == (2, 32, 32)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("orientation", [1, 2, 3, 4, 5, 6, 7, 8])
def test_write_to_buffer_matches_reference_packing(dec, oracle, dtype, orientation):
    """ImageStream::write_to_buffer on the device: interleave + u8/u16 rounding + all 8 orientations."""
    data = fixture_bytes("alpha_premultiplied", "input.jxl")  # RGBA, non-square
    dec.decode(data)
    got = dec.frame_to_buffer(0, dtype, orientation)
    img = oracle.OracleImage(data, threads=4)
    want = img.frame_to_buffer(0, dtype, orientation)
    assert got.shape == want.shape and got.shape[2] == 4
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_write_to_buffer_mixes_spot_colours(dec, oracle, dtype):
    """Spot-colour channels blended into RGB by the packing kernel, alpha appended (fb.rs:246-283, 335-362)."""
    data = fixture_bytes("spot", "input.jxl")
    dec.decode(data)
    got = dec.frame_to_buffer(0, dtype, 6)
    want = oracle.OracleImage(data, threads=4).frame_to_buffer(0, dtype, 6)
    assert got.shape == want.shape == (600, 400, 4)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    dec.release_frames()


def test_original_icc_matches_oracle(dec, oracle):
    """The product's host side reconstructs the embedded ICC profile (shared code path with the oracle)."""
    data = fixture_bytes("spot", "input.jxl")
    dec.decode(data)
    assert dec.original_icc() == oracle.OracleImage(data, threads=2).original_icc() != b""
    dec.release_frames()


def test_blend_modes_and_swapped_patch_roles(dec):
    """blend_single (blend.rs:550-727) incl. the *Below patch modes: the kernel against the formulas in f32 numpy
    (each expression is a chain of single IEEE operations, so numpy reproduces it bit for bit)."""
    import itertools
    import torch
    rng = np.random.default_rng(3)
    shape = (33, 47)
    f32 = np.float32
    base0, patch, ba, na = [rng.uniform(-0.2, 1.2, size=shape).astype(f32) for _ in range(4)]
    one = f32(1.0)
    for mode, clamp, premultiplied, swapped in itertools.product((4, 5, 6), (False, True), (False, True), (False, True)):
        t = [torch.from_numpy(x.copy()).cuda() for x in (base0, patch, ba, na)]
        dec.blend(t[0], t[1], t[2], t[3], mode, clamp, premultiplied, swapped)
        dec.sync()
        got = t[0].cpu().numpy()
        b, n = (patch, base0) if swapped else (base0, patch)
        if mode == 6:
            nn = np.clip(n, 0, 1).astype(f32) if clamp else n
            want = b + nn * (one - b)
        else:
            b_a, n_a = (na, ba) if swapped else (ba, na)
            n_a = np.clip(n_a, 0, 1).astype(f32) if clamp else n_a
            if mode == 5:
                want = b + n_a * n
            elif premultiplied:
                want = n + b * (one - n_a)
            else:
                mixed = one - (one - n_a) * (one - b_a)
                with np.errstate(divide="ignore"):
                    recip = np.where(mixed > 0, one / mixed, f32(0)).astype(f32)
                want = (n_a * n + b_a * b * (one - n_a)) * recip
        assert np.array_equal(got.view(np.uint32), want.astype(f32).view(np.uint32)), (mode, clamp, premultiplied, swapped)


def test_mutated_streams_end_in_values(dec):
    """Bit flips / truncations / overwritten runs in valid streams: every decode ends in pixels or a
    JxlError value, and the decoder keeps working (tools/mutate_check.py runs the same under
    compute-sanitizer memcheck)."""
    import random
    import jxl_oxide_b200
    rng = random.Random(99)
    for name in ("opsin_inverse", "grayalpha", "upsampling", "cafe", "delta_palette", "spot", "animation_spline", "grayscale"):
        data = fixture_bytes(name, "input.jxl")
        for i in range(12):
            m = bytearray(data)
            if i % 3 == 0:
                pos = rng.randrange(min(40, len(m) // 4), len(m))
                m[pos] ^= 1 << rng.randrange(8)
            elif i % 3 == 1:
                m = m[: rng.randrange(len(m) // 8, len(m))]
            else:
                pos = rng.randrange(len(m) // 3, len(m) - 8)
                for k in range(8):
                    m[pos + k] = rng.randrange(256)
            try:
                dec.decode(bytes(m))
                dec.release_frames()
            except jxl_oxide_b200.JxlError as e:
                assert e.code in (1, 2, 3, 6)
        dec.decode(data)
        dec.release_frames()


def test_animation_all_frames_bit_exact(dec, oracle):
    """Multi-frame codestream with cropped, blended frames and reference slots: every displayed frame."""
    data = fixture_bytes("animation_icos4d", "input.jxl")
    dec.decode(data)
    img = oracle.OracleImage(data, threads=8)
    assert dec.num_frames() == img.num_frames == 48
    for k in range(img.num_frames):
        got = dec.frame_planar(k)
        want = img.frame(k)[0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), k
    dec.release_frames()


def test_animation_splines_bit_exact(dec, oracle):
    """Spline rendering: the host-built arc list splatted by splat_splines_kernel, all 60 frames against the oracle."""
    data = fixture_bytes("animation_spline", "input.jxl")
    dec.decode(data)
    img = oracle.OracleImage(data, threads=8)
    assert dec.num_frames() == img.num_frames == 60
    for k in range(img.num_frames):
        got = dec.frame_planar(k)
        want = img.frame(k)[0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), k
    dec.release_frames()
