"""Splines and noise on upsampled VarDCT frames (tools/synth_enc.cc --upsampling / --noise / --splines).

The reference renders both on the coded-resolution grid, before upsampling (jxl-render/src/render.rs:136-149): splines
keep their frame coordinates and are clipped to the coded planes (features/spline.rs:180-251); the noise field is built
at the upsampled frame size, with that size's groups, seeds and mirroring, and its top-left coded-size part is added
(features/noise.rs:12-110). Checked here on the oracle: the noise stage against a numpy restatement of init_noise and
render_noise, the splines stage against the same splines drawn on a frame coded at full size, and the order against the
float64 upsampling model of tests/filter_model.py."""
import os
import subprocess

import numpy as np
import pytest

import bench
import filter_model as fm

# (width, height, k): every width but 1000 is not a multiple of k; 7x5 at k = 8 is coded as 1x1
FRAMES = [(w, h, k) for (w, h) in [(7, 5), (130, 70), (257, 256), (1000, 600)] for k in (2, 4, 8)]
ERR_BITSTREAM, ERR_UNSUPPORTED = 1, 2


def encode(tmp_path, w, h, args, seed=1):
    path = str(tmp_path / f"f_{w}x{h}_{seed}_{'_'.join(args).replace('-', '')}.jxl")
    if not os.path.exists(path):
        subprocess.check_call([bench.synth_tool(), "--width", str(w), "--height", str(h), "--seed", str(seed), "-o", path] +
                              list(args), stderr=subprocess.DEVNULL)
    return open(path, "rb").read()


def up_args(k, *more):
    return (["--upsampling", str(k)] if k != 1 else []) + list(more)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ---- numpy restatement of features/noise.rs ----

M64 = (1 << 64) - 1


def _split_mix(z):  # noise.rs:454-458, on uint64 arrays
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def noise_field(width, height, group_dim, seed0):
    """init_noise's random planes (before the high-pass): per group, eight xorshift128+ streams seeded by seed0 and the
    group origin, batches of 16 floats in [1, 2) filled channel after channel (noise.rs:88-160, 199-235, 405-451)."""
    field = np.zeros((3, height, width), dtype=np.float32)
    with np.errstate(over="ignore"):
        for y0 in range(0, height, group_dim):
            for x0 in range(0, width, group_dim):
                gw, gh = min(group_dim, width - x0), min(group_dim, height - y0)
                s0 = np.empty(8, np.uint64)
                s1 = np.empty(8, np.uint64)
                s0[0] = _split_mix(np.uint64((seed0 + 0x9E3779B97F4A7C15) & M64))
                s1[0] = _split_mix(np.uint64((((x0 << 32) + y0) + 0x9E3779B97F4A7C15) & M64))
                for i in range(1, 8):
                    s0[i], s1[i] = _split_mix(s0[i - 1]), _split_mix(s1[i - 1])
                wn2 = -(-gw // 16)
                out = np.empty((3 * gh * wn2, 8), np.uint64)
                for step in range(out.shape[0]):
                    a, b = s0, s1
                    out[step] = a + b
                    s0 = b
                    a = a ^ (a << np.uint64(23))
                    s1 = a ^ (b ^ (a >> np.uint64(18)) ^ (b >> np.uint64(5)))
                lo = (out & np.uint64(0xFFFFFFFF)).astype(np.uint32)
                hi = (out >> np.uint64(32)).astype(np.uint32)
                words = np.stack([lo, hi], -1).reshape(3, gh, wn2 * 16)  # lane i gives floats 2i and 2i + 1
                vals = ((words >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32)
                field[:, y0:y0 + gh, x0:x0 + gw] = vals[:, :, :gw]
    return field


def _mirror(p, n):
    return np.where(p < 0, -p - 1, np.where(p >= n, 2 * n - p - 1, p))


def render_noise(xyb, field, group_dim, lut8, corr_x=0.0, corr_b=1.0):
    """render_noise (noise.rs:12-86) on the planes `xyb` (the top-left part of the field's frame), float32 throughout,
    with the 5x5 high-pass of init_noise: rows added in the order of its 5-row ring buffer (noise.rs:297-320), mirrored
    at the field's edges."""
    f32 = np.float32
    _, fh, fw = field.shape
    h, w = xyb[0].shape
    ys, xs = np.arange(h)[:, None], np.arange(w)[None, :]
    ly = ys % group_dim
    n = []
    for c in range(3):
        acc = np.zeros((h, w), np.float32)
        for s in range(5):
            r = ly - 2 + ((s - ly) % 5 + 5) % 5
            sy = _mirror(ys - ly + r, fh)
            for dx in range(5):
                sx = _mirror(xs + dx - 2, fw)
                acc = acc + field[c][sy, sx] * f32(0.16)
        n.append(acc - field[c][:h, :w] * f32(4.0))
    lut = np.array(list(lut8) + [lut8[7]], np.float32)
    gx, gy, gb = (p.astype(np.float32) for p in xyb)
    in_x, in_y = gx + gy, gy - gx

    def strength(v):
        scaled = np.maximum(f32(0.0), v * f32(3.0))
        i = np.minimum(np.nan_to_num(scaled, nan=0.0).astype(np.int64), 7)
        frac = scaled - i.astype(np.float32)
        return (lut[i + 1] - lut[i]) * frac + lut[i]
    sx, sy = strength(in_x), strength(in_y)
    nx = f32(0.22) * sx * (f32(0.0078125) * n[0] + f32(0.9921875) * n[2])
    ny = f32(0.22) * sy * (f32(0.0078125) * n[1] + f32(0.9921875) * n[2])
    nsum = nx + ny
    return [gx + (f32(corr_x) * nsum + nx - ny), gy + nsum, gb + f32(corr_b) * nsum]


def noise_lut(seed):
    """The LUT tools/synth_enc.cc --noise writes (write_features): 64 + mt19937() % 512 per entry, over 1024."""
    rng = np.random.RandomState()  # numpy's MT19937 with the same init_genrand as std::mt19937
    rng.seed((seed ^ 0x6E015E00) & 0xFFFFFFFF)
    return [np.float32((64 + int(rng.randint(0, 1 << 32, dtype=np.uint64)) % 512) / 1024) for _ in range(8)]


# ---- tests ----

@pytest.mark.parametrize("w,h,k", FRAMES)
def test_all_zero_noise_lut_changes_nothing(oracle, tmp_path, w, h, k):
    """With an all-zero LUT the noise adds exact zeros: the frame decodes bit for bit as without noise."""
    plain = oracle.OracleImage(encode(tmp_path, w, h, up_args(k)), threads=8).frame(0)[0]
    img = oracle.OracleImage(encode(tmp_path, w, h, up_args(k, "--noise-zero")), threads=8, capture=True)
    got = img.frame(0)[0]
    assert got.shape == (3, h, w)
    assert np.array_equal(bits(got), bits(plain))
    assert [p.shape for p in img.stage("noise")] == [(-(-h // k), -(-w // k))] * 3


@pytest.mark.parametrize("w,h,k", [(7, 5, 8), (130, 70, 2), (257, 256, 4), (257, 256, 8), (1000, 600, 2), (1000, 600, 8)])
def test_noise_stage_matches_model(oracle, tmp_path, w, h, k):
    img = oracle.OracleImage(encode(tmp_path, w, h, up_args(k, "--noise")), threads=8, capture=True)
    before, got = img.stage("epf"), img.stage("noise")
    cw, ch = -(-w // k), -(-h // k)
    assert [p.shape for p in got] == [(ch, cw)] * 3
    lut, seed0 = noise_lut(1), 1 << 32  # the image's first shown frame
    want = render_noise(before, noise_field(w, h, 256, seed0), 256, lut)
    for g, wv in zip(got, want):
        assert np.array_equal(bits(g), bits(wv))
    assert max(np.abs(g - b).max() for g, b in zip(got, before)) > 1e-3, "the noise left the planes as they were"
    # planted error: the field built at the coded size
    wrong = render_noise(before, noise_field(cw, ch, 256, seed0), 256, lut) if min(cw, ch) >= 2 else None
    if wrong is not None:
        assert any(not np.array_equal(bits(g), bits(x)) for g, x in zip(got, wrong))
    # the final frame is the noisy coded grid upsampled (features before upsampling)
    up, up_bound = fm.upsample(np.stack(got).astype(np.float64)[0], k)
    plane = img.stage("upsampled")[0].astype(np.float64)
    assert (np.abs(plane - up[:h, :w]) <= up_bound[:h, :w] + 1e-6).all()


@pytest.mark.parametrize("w,h,k", [(130, 70, 2), (257, 256, 4), (1000, 600, 8), (1000, 600, 2), (7, 5, 8)])
def test_splines_stage_is_the_full_size_rendering_on_the_coded_grid(oracle, tmp_path, w, h, k):
    """The spline list depends on the seed and the frame size only, so a frame of the same size coded at full resolution
    draws the same arcs; what they add there, restricted to the coded grid at the same (unscaled) coordinates, is what
    they add to the upsampled frame's coded planes. Some splines start right of the coded width and are clipped."""
    n = 1 if w * h < 100 else 6
    full = oracle.OracleImage(encode(tmp_path, w, h, ["--splines", str(n)]), threads=8, capture=True)
    img = oracle.OracleImage(encode(tmp_path, w, h, up_args(k, "--splines", str(n))), threads=8, capture=True)
    cw, ch = -(-w // k), -(-h // k)
    d_full = np.stack(full.stage("splines")).astype(np.float64) - np.stack(full.stage("epf"))
    d_up = np.stack(img.stage("splines")).astype(np.float64) - np.stack(img.stage("epf"))
    assert d_up.shape == (3, ch, cw)
    assert np.abs(d_up).max() > 1e-3, "no spline reached the coded planes"
    tol = 1e-5 * (1 + np.abs(d_full[:, :ch, :cw]))
    assert (np.abs(d_up - d_full[:, :ch, :cw]) <= tol).all(), np.abs(d_up - d_full[:, :ch, :cw]).max()
    if w * h >= 100:
        # planted error: coordinates scaled by k (the full-size rendering sampled every k-th pixel)
        assert np.abs(d_up - d_full[:, ::k, ::k][:, :ch, :cw]).max() > 1e-3
        # planted error: splines added after upsampling instead of before
        pre = np.stack(img.stage("epf")).astype(np.float64)
        plane = img.stage("upsampled")[1].astype(np.float64)
        after, bound = fm.upsample(pre[1], k)
        after = after[:h, :w] + d_full[1]
        right, rbound = fm.upsample(pre[1] + d_up[1], k)
        assert (np.abs(plane - right[:h, :w]) <= rbound[:h, :w] + 1e-5).all()
        assert (np.abs(plane - after) > bound[:h, :w] + 1e-3).any()


@pytest.mark.parametrize("k", [2, 4, 8])
def test_splines_and_noise_together(oracle, tmp_path, k):
    """Noise goes on after the splines, from the splines stage."""
    w, h = 1000, 600
    img = oracle.OracleImage(encode(tmp_path, w, h, up_args(k, "--splines", "6", "--noise")), threads=8, capture=True)
    want = render_noise(img.stage("splines"), noise_field(w, h, 256, 1 << 32), 256, noise_lut(1))
    for g, wv in zip(img.stage("noise"), want):
        assert np.array_equal(bits(g), bits(wv))
    assert img.frame(0)[0].shape == (3, h, w)


def test_noise_needs_a_frame_of_two_samples(oracle, tmp_path):
    """The mirror runs over the frame, so a 1x1 frame is refused and a 7x5 one coded at 1x1 is not."""
    assert oracle.OracleImage(encode(tmp_path, 1, 1, up_args(2))).frame(0)[0].shape == (3, 1, 1)
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(encode(tmp_path, 1, 1, up_args(2, "--noise")))
    assert e.value.code == ERR_UNSUPPORTED
    assert oracle.OracleImage(encode(tmp_path, 7, 5, up_args(8, "--noise"))).frame(0)[0].shape == (3, 5, 7)


@pytest.mark.parametrize("feature", [["--noise"], ["--splines", "2"], ["--noise", "--splines", "2"]])
def test_patches_with_upsampling_and_features_are_refused(oracle, tmp_path, feature):
    """Patches are blended after upsampling, splines and noise before it: together they are refused before the patch is
    looked at. The same patch on its own reaches blending, which fails on its missing reference frame."""
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(encode(tmp_path, 130, 70, up_args(2, "--dangling-patch", *feature)))
    assert e.value.code == ERR_UNSUPPORTED and "together with patches on an upsampled frame" in str(e.value)
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(encode(tmp_path, 130, 70, up_args(2, "--dangling-patch")))
    assert e.value.code == ERR_BITSTREAM and "reference frame that was not decoded" in str(e.value)


def test_frames_without_upsampling_keep_their_order(oracle, tmp_path):
    """Upsampling 1: splines and noise on the full-size planes with a field of their size, as before."""
    w, h = 257, 130
    img = oracle.OracleImage(encode(tmp_path, w, h, ["--splines", "3", "--noise"]), threads=8, capture=True)
    want = render_noise(img.stage("splines"), noise_field(w, h, 256, 1 << 32), 256, noise_lut(1))
    for g, wv in zip(img.stage("noise"), want):
        assert np.array_equal(bits(g), bits(wv))
    assert img.stage("upsampled") == []
