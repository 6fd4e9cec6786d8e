"""GPU tests of the filter and colour chain on small, narrow and odd-width frames, and of the stage entry points against the
float64 / exact models of tests/filter_model.py.

launch_filters_fused (kernels/filters_fused.cu) picks its code path from the frame's geometry and filter settings. The
strip rectangle (fstrip::strip_rect) is empty unless width >= 128 and height >= 96, and the strip kernel needs a width that
is a multiple of 4, Gaborish and EPF 1 or 2. The shapes below reach:
  * stage-by-stage kernels (width or height < 16): 1x9, 9x1, 7x5, 15x15, 15x40, 40x15, 257x9;
  * the general fused kernel over the whole frame, TMA loads: 16x16, 17x19, 31x33, 63x40, 64x32, 68x36, 92x56, 120x48,
    124x100 (no strip rectangle), the odd widths 65x33, 66x70, 67x25, 1001x601, 257x256, 1002x258 (width % 4 != 0), and
    every shape with EPF 0 / 3 or Gaborish off;
  * the strip kernel for the interior plus the general kernel on the border tiles: 128x96, 132x100, 196x104, 256x256,
    256x257 with Gaborish and EPF 1 or 2 (the last tile column is pulled back whenever the rectangle's width is not a
    multiple of 56 columns, as in all of these);
  * the general kernel with plain global loads instead of TMA (a plane pitch that is not a multiple of 16 bytes): Modular
    frames with restoration filters at odd widths, at least 16 x 16.
Which of the stage kernels or the fused kernel ran is checked on the device with the decoder's launch profile.
"""
import itertools

import numpy as np
import pytest

import bench
import filter_model as fm
from test_gpu_parity import _check_vardct, _decode_both

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

UNDER16 = [(1, 9), (9, 1), (7, 5), (15, 15), (15, 40), (40, 15)]
GENERAL = [(16, 16), (17, 19), (31, 33), (63, 40)]
STRIP = [(64, 32), (68, 36), (92, 56), (120, 48), (124, 100), (128, 96), (132, 100), (196, 104)]
ODD = [(65, 33), (66, 70), (67, 25), (1001, 601)]
EDGES = [(256, 256), (256, 257), (257, 256), (257, 9), (1002, 258)]
CONFIGS = [(0, True), (1, True), (2, True), (3, True), (0, False), (2, False)]  # (EPF iterations, Gaborish)
LARGE = {(1001, 601), (1002, 258)}


def synth(w, h, iters=2, gaborish=True, extra=()):
    ex = ("--sharpness-cell", "1") + (("--epf-iters", str(iters)) if iters != 2 else ()) + (() if gaborish else ("--no-gaborish",))
    return bench.synth_frame(w, h, 3, extra=ex + tuple(extra))


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


CASES = [(s, c) for s in UNDER16 + GENERAL + STRIP + ODD + EDGES for c in CONFIGS if s not in LARGE or c in ((2, True), (3, True))]


@pytest.mark.parametrize("size,config", CASES, ids=[f"{s[0]}x{s[1]}-epf{c[0]}{'' if c[1] else '-nogab'}" for s, c in CASES])
def test_small_frames_bit_exact(dec, oracle, size, config):
    """Fused and stage by stage against the oracle, bit for bit (the EPF sigma grid included)."""
    data = synth(*size, iters=config[0], gaborish=config[1])
    _check_vardct(dec, oracle, data)
    filtered = config[0] > 0 or config[1]  # with neither filter no filter kernel runs
    assert (fused_launches(dec, data) > 0) == (filtered and min(size) >= 16)


def fused_launches(dec, data):
    """Launches of the fused filter kernels in a decode with filter fusion on (0: the stage-by-stage kernels ran)."""
    dec.set_fuse_filters(True)
    dec.set_profile(True)
    dec.profile_reset()
    try:
        dec.decode(data)
        return dec.profile("filters_fused")[0]
    finally:
        dec.set_profile(False)
        dec.release_frames()


@pytest.mark.parametrize("size", [(7, 5), (17, 19), (65, 33), (128, 96)])
@pytest.mark.parametrize("output_colour", [1, 2])
def test_small_frames_other_output_encodings(dec, oracle, size, output_colour):
    dec.set_fuse_filters(True)
    got, want, _ = _decode_both(dec, oracle, synth(*size), output_colour=output_colour)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("size", [(15, 40), (67, 25), (128, 96)])
def test_small_frames_enum_target(dec, oracle, size):
    _check_vardct(dec, oracle, synth(*size, extra=("--colour", "p3")))


@pytest.mark.parametrize("size,sigma,iters", [((301, 67), 1.0, 3), ((257, 9), 0.3, 2), ((513, 20), 2.5, 1), ((259, 260), 1.0, 2)])
def test_modular_frames_with_filters_plain_loads(dec, oracle, size, sigma, iters):
    """Modular frames with Gaborish + EPF (constant sigma) at odd widths: planes whose pitch is not a multiple of 16 bytes,
    which encode_plane_maps refuses to describe, so the fused kernel (the output planes keep the input's pitch) runs with
    plain global loads. 257 x 9 is under 16 high and goes to the stage kernels instead."""
    data = bench.synth_frame(size[0], size[1], 3, extra=("--modular", "--modular-filters", str(sigma), "--epf-iters", str(iters)))
    for fused in (True, False):
        dec.set_fuse_filters(fused)
        got, want, _ = _decode_both(dec, oracle, data)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), fused
        _, stride = dec.frame_channel_device(0, 0)
        assert (stride * 4) % 16 != 0, "the frame's planes would take the TMA path"
    assert (fused_launches(dec, data) > 0) == (min(size) >= 16)


def test_pipeline_mixes_small_and_large_frames(oracle):
    import ctypes
    import jxl_oxide_b200 as J
    datas = [synth(*s) for s in [(1, 9), (9, 1), (17, 19), (65, 33), (124, 100), (257, 9)]] + [bench.synth_frame(2000, 1500, 3)]
    datas += [synth(67, 25, iters=3), synth(64, 32, gaborish=False)]
    want = []
    for d in datas:
        img = oracle.OracleImage(d, threads=8)
        want.append(img.frame(0)[0])
        img.close()
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for i, d in enumerate(datas):
            p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=i)
        seen = set()
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            w = want[tag]
            assert nbytes == w.nbytes
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=np.float32).reshape(w.shape).copy()
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint32), w.view(np.uint32)), tag
            seen.add(tag)
        assert seen == set(range(len(datas)))
    finally:
        p.close()


# ---- stage entry points on synthetic planes against the models ----

PLANE_SHAPES = [(w, h) for w in range(1, 10) for h in range(1, 10)] + [(16, 16), (17, 19), (65, 33), (128, 96), (257, 9)]


def _device(planes, extra_cols):
    """Device planes with a row stride of width + extra_cols floats."""
    import torch
    out = []
    for p in planes:
        h, w = p.shape
        t = torch.full((h, w + extra_cols), float("nan"), dtype=torch.float32, device="cuda")
        t[:, :w] = torch.from_numpy(np.ascontiguousarray(p))
        out.append(t[:, :w])
    return out


def _ratio(got, want, bound):
    return float(np.max(np.abs(got.astype(np.float64) - want) / np.maximum(bound, 1e-300)))


def random_planes(w, h, seed, amp=0.02):
    rng = np.random.default_rng(seed)
    base = rng.uniform(-amp, amp, size=(3, h, w)) + np.array([0.01, 0.5, 0.4])[:, None, None]
    return [base[c].astype(np.float32) for c in range(3)]


def test_gaborish_entry_point(dec):
    wts = [[0.115169525, 0.061248592], [0.2, 0.05], [0.08, 0.12]]
    for i, (w, h) in enumerate(PLANE_SHAPES):
        planes = random_planes(w, h, i)
        t = _device(planes, 3 + i % 5)
        dec.gaborish(t, wts)
        dec.sync()
        for c in range(3):
            m, b = fm.gaborish(planes[c], float(np.float32(wts[c][0])), float(np.float32(wts[c][1])))
            assert _ratio(t[c].cpu().numpy(), m, b) <= 1.0, (w, h, c)


def test_epf_entry_point(dec):
    import torch
    import jxl_oxide_b200 as J
    sigmas = np.array([0.0, 0.29999998, 0.3, 0.30000001, 0.45, 1.0, 2.5], dtype=np.float32)
    for i, (w, h) in enumerate(PLANE_SHAPES):
        rng = np.random.default_rng(i + 1000)
        grid = rng.choice(sigmas, size=((h + 7) // 8, (w + 7) // 8)).astype(np.float32)
        grid.flat[0] = np.float32(0.3)
        for iters, constant in itertools.product((0, 1, 2, 3), (False, True)):
            planes = random_planes(w, h, i)
            t = _device(planes, 1 + i % 4)
            prm = J.EpfParams(iters, (40.0, 5.0, 3.5), 0.9, 6.5, 2.0 / 3.0, 0.75)
            sg = None
            if not constant:
                sg = torch.zeros((grid.shape[0], grid.shape[1] + 2), dtype=torch.float32, device="cuda")
                sg[:, :grid.shape[1]] = torch.from_numpy(grid)
                sg = sg[:, :grid.shape[1]]
            dec.epf(t, sg, prm)
            dec.sync()
            got = [x.cpu().numpy() for x in t]
            if iters == 0:
                assert all(np.array_equal(g.view(np.uint32), p.view(np.uint32)) for g, p in zip(got, planes)), (w, h)
                continue
            sigma = fm.sigma_per_pixel(None if constant else grid, h, w, 0.75)
            m, b = fm.epf(planes, sigma, iters)
            for c in range(3):
                assert _ratio(got[c], m[c], b[c]) <= 1.0, (w, h, iters, constant, c)


def test_xyb_to_rgb_entry_point(dec):
    from test_filter_model import srgb_approx_rel
    ob = [fm.OPSIN_BIAS] * 3
    mat = [float(v) for v in fm.OPSIN_INV.ravel()]
    for i, (w, h) in enumerate(PLANE_SHAPES[::7]):
        rng = np.random.default_rng(i)
        xyb = [rng.uniform(-0.03, 0.03, (h, w)).astype(np.float32), rng.uniform(0.0, 0.9, (h, w)).astype(np.float32),
               rng.uniform(0.0, 0.9, (h, w)).astype(np.float32)]
        lin, lb = fm.xyb_to_linear(xyb)
        for srgb_tf in (0, 1):
            t = _device(xyb, 2)
            dec.xyb_to_rgb(t, ob, mat, 255.0, srgb_tf)
            dec.sync()
            for c in range(3):
                m, b = fm.srgb(lin[c], lb[c], srgb_approx_rel()) if srgb_tf else (lin[c], lb[c])
                assert _ratio(t[c].cpu().numpy(), m, b) <= 1.0, (w, h, srgb_tf, c)


@pytest.mark.parametrize("factor", [2, 4, 8])
def test_upsample_entry_point(dec, factor):
    """jxlb_upsample on every shape up to 9 x 9 (one-sample-wide and -high inputs take the reference's in-place padding
    quirk) with a row stride larger than the width: within the float64 bound, and bit for bit the oracle's."""
    import torch
    from test_filter_model import UPSAMPLE_SHAPES, oracle_upsample
    rng = np.random.default_rng(factor)
    for i, (w, h) in enumerate(UPSAMPLE_SHAPES):
        x = rng.uniform(-0.2, 1.2, (h, w)).astype(np.float32)
        src = torch.full((h, w + 1 + i % 5), float("nan"), dtype=torch.float32, device="cuda")
        src[:, :w] = torch.from_numpy(x)
        got = dec.upsample(src[:, :w], factor)
        dec.sync()
        got = got.cpu().numpy()
        m, b = fm.upsample(x, factor)
        assert _ratio(got, m, b) <= 1.0, (factor, w, h)
        assert np.array_equal(got.view(np.uint32), oracle_upsample(x, factor).view(np.uint32)), (factor, w, h)


# ---- exact integer stages ----

I32 = np.iinfo(np.int32)


def _extreme_ints(rng, shape):
    v = rng.integers(I32.min, I32.max, size=shape, dtype=np.int64, endpoint=True)
    pick = rng.integers(0, 4, size=shape)
    v = np.where(pick == 0, I32.max - rng.integers(0, 3, size=shape), v)
    v = np.where(pick == 1, I32.min + rng.integers(0, 3, size=shape), v)
    return v.astype(np.int32)


def test_rct_inverse_all_variants_at_int32_limits(dec):
    import torch
    rng = np.random.default_rng(11)
    for rct_type in range(42):
        a, b, c = [_extreme_ints(rng, (5, 37)) for _ in range(3)]
        t = [torch.from_numpy(x.copy()).cuda() for x in (a, b, c)]
        dec.rct_inverse(t, rct_type)
        dec.sync()
        for got, want in zip(t, fm.rct_inverse(a, b, c, rct_type)):
            assert np.array_equal(got.cpu().numpy(), want), rct_type


@pytest.mark.parametrize("horizontal", [True, False])
def test_squeeze_inverse_edges_and_int32_limits(dec, horizontal):
    import torch
    rng = np.random.default_rng(5)
    for n_avg, res_kind, lines, extreme in itertools.product((1, 2, 5, 8), ("same", "one_less"), (1, 3), (False, True)):
        n_res = n_avg if res_kind == "same" else n_avg - 1
        gen = (lambda s: _extreme_ints(rng, s)) if extreme else (lambda s: rng.integers(-300, 300, size=s).astype(np.int32))
        avg, res = gen((lines, n_avg)), gen((lines, n_res))
        want = fm.squeeze_inverse_h(avg, res)
        if not horizontal:
            avg, res, want = avg.T.copy(), res.T.copy(), want.T.copy()
        ta, tr = torch.from_numpy(avg).cuda(), torch.from_numpy(res).cuda()
        out = torch.zeros(want.shape, dtype=torch.int32, device="cuda")
        dec.squeeze_inverse(ta, tr, out, horizontal)
        dec.sync()
        assert np.array_equal(out.cpu().numpy(), want), (n_avg, res_kind, lines, extreme)


def test_blend_replace_add_mul(dec):
    """blend_single (blend.rs:550-605) modes 1-3 with and without clamp, in f32 numpy (single IEEE operations)."""
    import torch
    rng = np.random.default_rng(4)
    base0, patch = [rng.uniform(-0.3, 1.3, size=(19, 23)).astype(np.float32) for _ in range(2)]
    for mode, clamp in itertools.product((1, 2, 3), (False, True)):
        t = [torch.from_numpy(x.copy()).cuda() for x in (base0, patch)]
        dec.blend(t[0], t[1], None, None, mode, clamp)
        dec.sync()
        if mode == 1:
            want = patch
        elif mode == 2:
            want = base0 + patch
        else:
            want = base0 * (np.clip(patch, 0, 1).astype(np.float32) if clamp else patch)
        assert np.array_equal(t[0].cpu().numpy().view(np.uint32), want.astype(np.float32).view(np.uint32)), (mode, clamp)
