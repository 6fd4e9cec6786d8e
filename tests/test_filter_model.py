"""The float64 models of tests/filter_model.py against the oracle, stage by stage, on small, narrow and odd-width frames.

Each stage's captured f32 input goes through the model, and the captured f32 output must lie within the model's error
bound everywhere. The negative controls plant known misreadings into the model and require the same comparison to fail,
which shows that the bounds are tight enough to catch such an error in the oracle or the kernels (they share the
oracle's stage order and are compared with it bit for bit on the GPU).
"""
import ctypes
import functools

import numpy as np
import pytest

import bench
import filter_model as fm
import oracle_lib
from conftest import fixture_bytes

F32 = np.float32

# (width, height) of the synthetic frames: under 16 (stage-by-stage kernels), the general fused kernel, a strip
# rectangle with the pulled-back last tile column, odd widths, partial 8x8 blocks and group edges
SMALL = [(1, 1), (9, 1), (1, 9), (7, 5), (15, 40), (17, 19), (31, 33), (64, 32), (65, 33), (67, 25)]
EDGES = [(256, 257), (257, 9)]


def synth(w, h, seed=3, extra=()):
    return bench.synth_frame(w, h, seed, extra=("--sharpness-cell", "1") + tuple(extra))


@functools.lru_cache(maxsize=1)
def srgb_approx_rel():
    """Largest relative distance of the kernels' sRGB curve (pixel_math.cuh, host build) from the exact curve, on the
    linear segment and above it, over every f32 in [2^-16, 32): the approximation is a polynomial in the mantissa times a
    per-binade factor, so a complete sweep of the binades the samples occupy bounds it (values below 2^-16 lie on the
    linear segment, whose relative error does not depend on the magnitude)."""
    L = oracle_lib.emu_lib()
    L.jxle_linear_to_srgb.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    worst = [0.0, 0.0]
    for e in range(-16, 5):
        bits = np.arange(0, 1 << 23, dtype=np.uint32) + np.uint32((e + 127) << 23)
        v = bits.view(np.float32)
        got = np.empty_like(v)
        L.jxle_linear_to_srgb(v.ctypes.data, got.ctypes.data, v.size)
        want = fm.srgb_exact(v.astype(np.float64))
        rel = np.abs(got - want) / want
        lin = v <= F32(fm.SRGB_THRESHOLD)
        for k, sel in enumerate((lin, ~lin)):
            if sel.any():
                worst[k] = max(worst[k], float(rel[sel].max()))
    return tuple(worst)


def _ratio(got, want, bound):
    return float(np.max(np.abs(got.astype(np.float64) - want) / np.maximum(bound, 1e-300)))


def chain_ratios(data, gab_swap=False, faults=None, srgb_slope=12.92, modular_sigma=None, colour=True):
    """{stage: worst |oracle - model| / bound} over the stages the frame runs (> 1: outside the bound)."""
    img = oracle_lib.OracleImage(data, threads=4, capture=True)
    _, iters = img.frame_filters(0)
    pre, gab, epf, rgb = img.stage("pre_filter"), img.stage("gaborish"), img.stage("epf"), img.stage("rgb")
    out = {}
    src = pre
    if gab:
        r = 0.0
        for c in range(3):
            m, b = fm.gaborish(pre[c], *fm.GAB_DEFAULT, swap_weights=gab_swap)
            r = max(r, _ratio(gab[c], m, b))
        out["gaborish"] = r
        src = gab
    if epf:
        h, w = src[0].shape
        sig = img.stage("epf_sigma")
        sigma = fm.sigma_per_pixel(sig[0] if sig else None, h, w, modular_sigma)
        m, b = fm.epf(src, sigma, iters, faults=faults)
        out["epf"] = max(_ratio(epf[c], m[c], b[c]) for c in range(3))
        src = epf
    plain = not any(img.stage(s) for s in ("upsampled", "patches", "splines", "noise"))
    if colour and rgb and len(rgb) == 3 and plain and img.xyb:
        lin, lb = fm.xyb_to_linear(src)
        r = 0.0
        for c in range(3):
            assert np.abs(lin[c]).max() < 32.0, "outside the swept range of the sRGB bound"
            m, b = fm.srgb(lin[c], lb[c], srgb_approx_rel(), slope=srgb_slope)
            r = max(r, _ratio(rgb[c], m, b))
        out["rgb"] = r
    img.close()
    return out


def frame(w, h, iters=2, gaborish=True, seed=3):
    extra = ("--epf-iters", str(iters)) if iters != 2 else ()
    if not gaborish:
        extra += ("--no-gaborish",)
    return synth(w, h, seed, extra)


def modular_frame(w, h, sigma, iters, seed=3):
    return bench.synth_frame(w, h, seed, extra=("--modular", "--modular-filters", str(sigma), "--epf-iters", str(iters)))


def _assert_within(ratios, stages):
    for s in stages:
        assert s in ratios, f"stage {s} did not run"
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f"oracle outside the float64 bound: {bad}"


@pytest.mark.parametrize("size", SMALL + EDGES)
@pytest.mark.parametrize("iters,gaborish", [(0, True), (1, True), (2, True), (3, True), (0, False), (2, False)])
def test_synthetic_frames_within_float64_bounds(size, iters, gaborish):
    ratios = chain_ratios(frame(*size, iters=iters, gaborish=gaborish))
    _assert_within(ratios, (["gaborish"] if gaborish else []) + (["epf"] if iters else []) + ["rgb"])


@pytest.mark.parametrize("name", ["opsin_inverse", "minecraft_vardct_e7", "grayscale", "alpha_premultiplied", "noise"])
def test_vardct_fixtures_within_float64_bounds(name):
    # libjxl's frames: their colour parameters are not the defaults the model assumes
    ratios = chain_ratios(fixture_bytes(name, "input.jxl"), colour=False)
    _assert_within(ratios, ["gaborish", "epf"])


@pytest.mark.parametrize("size,sigma,iters", [((301, 67), 1.0, 3), ((257, 9), 0.3, 2), ((513, 20), 2.5, 1)])
def test_modular_frames_with_filters_within_float64_bounds(size, sigma, iters):
    """Modular frames filter RGB samples with the constant sigma_for_modular (an f16 in the frame header)."""
    s16 = float(np.float16(sigma))
    ratios = chain_ratios(modular_frame(size[0], size[1], sigma, iters), modular_sigma=s16)
    _assert_within(ratios, ["gaborish", "epf"])


# ---- oracle filter stages on synthetic planes (all shapes up to 9 x 9, sigma grids straddling 0.3) ----

def _oracle_gaborish(planes, weights):
    L = oracle_lib.lib()
    L.jxlo_gaborish.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_uint32] * 2 + [ctypes.c_void_p]
    p = [np.ascontiguousarray(x, dtype=np.float32).copy() for x in planes]
    wt = np.asarray(weights, dtype=np.float32).ravel()
    L.jxlo_gaborish(*[x.ctypes.data for x in p], p[0].shape[1], p[0].shape[0], wt.ctypes.data)
    return p


def _oracle_epf(planes, sigma_grid, iters, sigma_const=1.0):
    L = oracle_lib.lib()
    L.jxlo_epf.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_uint32] * 2 + [ctypes.c_void_p, ctypes.c_float, ctypes.c_uint32]
    p = [np.ascontiguousarray(x, dtype=np.float32).copy() for x in planes]
    sg = None if sigma_grid is None else np.ascontiguousarray(sigma_grid, dtype=np.float32)
    L.jxlo_epf(*[x.ctypes.data for x in p], p[0].shape[1], p[0].shape[0], None if sg is None else sg.ctypes.data, sigma_const, iters)
    return p


SIGMAS = np.array([0.0, 0.29999998, 0.3, 0.30000001, 0.45, 1.0, 2.5], dtype=np.float32)


def random_planes(w, h, seed, amp=0.05):
    rng = np.random.default_rng(seed)
    base = rng.uniform(-amp, amp, size=(3, h, w)) + np.array([0.01, 0.5, 0.4])[:, None, None]
    return [base[c].astype(np.float32) for c in range(3)]


def sigma_grid(w, h, seed):
    rng = np.random.default_rng(seed + 1000)
    g = rng.choice(SIGMAS, size=((h + 7) // 8, (w + 7) // 8)).astype(np.float32)
    g.flat[0] = F32(0.3)  # exactly at the threshold: filtered (`< 0.3` copies)
    return g


PLANE_SHAPES = [(w, h) for w in range(1, 10) for h in range(1, 10)] + [(16, 16), (17, 19), (33, 9), (40, 15)]


def epf_plane_ratio(w, h, iters, constant=False, faults=None, seed=0, amp=0.002):
    # amp: small differences between neighbours, so that the EPF weights are not all zero at these sigmas
    planes = random_planes(w, h, seed, amp)
    grid = None if constant else sigma_grid(w, h, seed)
    got = _oracle_epf(planes, grid, iters, sigma_const=1.0)
    m, b = fm.epf(planes, fm.sigma_per_pixel(grid, h, w, 1.0), iters, faults=faults)
    return max(_ratio(got[c], m[c], b[c]) for c in range(3))


def test_oracle_filters_on_small_planes_within_float64_bounds():
    for i, (w, h) in enumerate(PLANE_SHAPES):
        planes = random_planes(w, h, i)
        wts = [[0.115169525, 0.061248592], [0.2, 0.05], [0.08, 0.12]]
        got = _oracle_gaborish(planes, wts)
        for c in range(3):
            m, b = fm.gaborish(planes[c], float(F32(wts[c][0])), float(F32(wts[c][1])))
            assert _ratio(got[c], m, b) <= 1.0, ("gaborish", w, h, c)
        for iters in (1, 2, 3):
            assert epf_plane_ratio(w, h, iters, seed=i) <= 1.0, ("epf", w, h, iters)
        assert epf_plane_ratio(w, h, 3, constant=True, seed=i) <= 1.0, ("epf constant sigma", w, h)


# ---- negative controls: each planted model error must put the oracle outside the bound ----

def test_negative_control_border_multiplier_column():
    r = chain_ratios(frame(65, 33, iters=3), faults=fm.EpfFaults(border_col=1))
    assert r["epf"] > 1.0


def test_negative_control_replicate_instead_of_mirror():
    r = chain_ratios(frame(17, 19, iters=3), faults=fm.EpfFaults(replicate=True))
    assert r["epf"] > 1.0
    assert max(epf_plane_ratio(w, h, 2, faults=fm.EpfFaults(replicate=True), seed=w * 9 + h) for w, h in [(3, 9), (9, 3), (2, 7)]) > 1.0


def test_negative_control_sigma_threshold_inclusive():
    # the sigma grids hold 0.3f exactly: filtered by the reference (`sigma < 0.3` copies), copied by the planted `<=`
    assert max(epf_plane_ratio(w, h, 1, faults=fm.EpfFaults(sigma_le=True), seed=i) for i, (w, h) in enumerate([(9, 9), (16, 16)])) > 1.0


def test_negative_control_swapped_gaborish_weights():
    assert chain_ratios(frame(17, 19, iters=0), gab_swap=True)["gaborish"] > 1.0
    assert chain_ratios(frame(9, 1, iters=0), gab_swap=True)["gaborish"] > 1.0


def test_negative_control_srgb_linear_slope():
    assert chain_ratios(frame(64, 32, iters=0), srgb_slope=12.9)["rgb"] > 1.0


def test_srgb_approximation_bound_is_small():
    # measured, not assumed: near u on the linear segment (the f32 threshold moves its end by an ulp), the polynomial's own error above it; both far below the
    # planted slope error (0.15 %)
    r_lin, r_pow = srgb_approx_rel()
    assert r_lin < 1e-5 and 0.0 < r_pow < 1e-3


def oracle_upsample(x, factor):
    L = oracle_lib.lib()
    L.jxlo_upsample.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty((x.shape[0] * factor, x.shape[1] * factor), dtype=np.float32)
    L.jxlo_upsample(x.ctypes.data, x.shape[1], x.shape[0], factor, out.ctypes.data)
    return out


UPSAMPLE_SHAPES = [(w, h) for w in range(1, 10) for h in range(1, 10)] + [(17, 3), (3, 17)]


@pytest.mark.parametrize("factor", [2, 4, 8])
def test_oracle_upsampling_within_float64_bounds(factor):
    """Every shape up to 9 x 9: one-sample-wide and one-sample-high inputs take the reference's in-place padding quirk."""
    rng = np.random.default_rng(factor)
    for w, h in UPSAMPLE_SHAPES:
        x = rng.uniform(-0.2, 1.2, (h, w)).astype(np.float32)
        m, b = fm.upsample(x, factor)
        assert _ratio(oracle_upsample(x, factor), m, b) <= 1.0, (factor, w, h)


def test_negative_control_upsampling_without_padding_quirk():
    # a proper mirror instead of the reference's in-place one differs on every one-sample-wide or -high input
    rng = np.random.default_rng(9)
    for factor in (2, 4, 8):
        for w, h in [(1, 5), (6, 1), (1, 2)]:
            x = rng.uniform(-0.2, 1.2, (h, w)).astype(np.float32)
            m, b = fm.upsample(x, factor, mirror_quirk=False)
            assert _ratio(oracle_upsample(x, factor), m, b) > 1.0, (factor, w, h)


def test_filter_launch_geometry_small_frames():
    """jxle_filter_geometry_check (tests/test_emu_filters.py) at every size from 16 x 16 to 130 x 130 and at the GPU test
    shapes: the strip rectangle and the border grid tile the frame exactly once."""
    L = oracle_lib.emu_lib()
    L.jxle_filter_geometry_check.restype = ctypes.c_int
    sizes = [(w, h) for w in range(16, 131) for h in range(16, 131)]
    sizes += [(64, 32), (68, 36), (92, 56), (120, 48), (124, 100), (128, 96), (65, 33), (66, 70), (67, 25), (1001, 601),
              (256, 256), (256, 257), (257, 256), (257, 9), (1002, 258)]
    for w, h in sizes:
        assert L.jxle_filter_geometry_check(w, h) == 0, (w, h)
