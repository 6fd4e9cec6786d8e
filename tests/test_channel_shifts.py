"""Channels coded below the frame's resolution: YCbCr Modular frames with chroma subsampling, and extra channels with
dim_shift or their own upsampling in Modular and VarDCT frames (tools/synth_enc.cc --ycbcr / --upsampling / --extra).

The oracle runs the same planner as the device, so the checks here do not go through it: the coded channels must equal
the encoder's own samples, and the final planes must lie within a float64 model's bound of the reference's arithmetic
(chroma upsampling and YCbCr -> RGB; the non-separable upsampling chain of tests/filter_model.py)."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

import bench
import filter_model as fm
from conftest import fixture_bytes

# bench.synth_frame(...) of the parent revision: the encoder's default output must not change
DIGESTS = [
    ((1000, 600, 7), (), 74283, "04cd6389b2cb0ef543e9cb7f6f60bd1d878981581af20dc76346adec8eba9eee"),
    ((600, 400, 3), ("--modular",), 226331, "a9f7e7beeef082b374f18bf72f1fd954805b9b72e51918892dd79e03eb9ff73f"),
    ((2600, 700, 5), (), 218700, "96869f369fd0ac584347809ea102d1d88ae8b7f1c8154e61c77cdb260632242c"),
    ((3840, 2160, 1), (), 970824, "95305433cd549370df652aa467f964f24f951ed79771564575fc451895da6521"),
    ((3840, 2160, 1), ("--modular",), 7869197, "e3f91d95ecaf26998cee773a763e384e3a8b228732d0d609141ea094ab1e0ffb"),
]

YCBCR = [(mode, w, h) for mode in ("444", "420", "422", "440") for (w, h) in [(300, 200), (257, 129), (5, 1), (1, 7), (1, 1), (513, 270)]]
# (upsampling, [TYPE:BITS:DIM_SHIFT:EC_UPSAMPLING ...], width, height): dim_shift 0-3 x ec_upsampling 1-8 against
# upsampling 1-8, total shift up to 6; a coded shift of 3 or more lands in the LF-group streams of a wide frame
EXTRA = [
    (1, ["alpha:8:1:1"], 300, 201),
    (1, ["alpha:8:2:1", "spot:12:0:1"], 600, 300),
    (1, ["unknown:10:3:1"], 2100, 900),
    (1, ["alpha:8:0:8", "unknown:8:3:8"], 2100, 333),
    (2, ["alpha:8:0:4", "spot:12:1:2"], 517, 301),
    (2, ["unknown:16:2:8"], 4200, 260),
    (4, ["alpha:8:2:4", "unknown:1:0:8"], 1030, 77),
    (8, ["alpha:8:3:8", "spot:10:0:8"], 4100, 37),
    (1, ["alpha:8:2:2"], 1, 1),
    (2, ["alpha:8:1:2"], 9, 1),
]
# VarDCT frames (upsampling 1): the extra channels ride in the GlobalModular, LF-group and pass-group streams
EXTRA_VARDCT = [
    (["alpha:8:2:1"], 600, 300),
    (["alpha:8:1:1", "unknown:12:3:8", "spot:10:0:2"], 2100, 900),
    (["alpha:8:0:4", "unknown:16:2:8"], 4200, 260),
    (["alpha:8:3:8"], 2600, 700),
    (["alpha:8:1:1"], 1, 1),
    (["spot:8:0:8", "alpha:8:1:2"], 257, 9),
]


def encode(tmp_path, w, h, args, seed=1, modular=True):
    """Encoded bytes and the --dump-raw samples (None where the frame has no channel coded without transforms)."""
    jxl, raw = str(tmp_path / "s.jxl"), str(tmp_path / "s.raw")
    if os.path.exists(raw):
        os.remove(raw)
    subprocess.check_call([bench.synth_tool()] + (["--modular"] if modular else []) +
                          ["--width", str(w), "--height", str(h), "--seed", str(seed), "-o", jxl, "--dump-raw", raw] + args,
                          stderr=subprocess.DEVNULL)
    return open(jxl, "rb").read(), np.fromfile(raw, dtype=np.int32) if os.path.exists(raw) else None


def extra_args(up, extras):
    out = ["--upsampling", str(up)] if up != 1 else []
    for e in extras:
        out += ["--extra", e]
    return out


def coded_equal(img, raw):
    coded = img.stage("modular_coded", np.int32)
    flat = np.concatenate([c.ravel() for c in coded])
    return coded, flat.size == raw.size and np.array_equal(flat, raw)


# ---- float64 models ----

def jpeg_upsample(x, hs, vs, w, h):
    """apply_jpeg_upsampling_single (jxl-render/src/filter/ycbcr.rs) in float64, cropped to w x h."""
    if hs:
        left = np.concatenate([x[:, :1], x[:, :-1]], 1)
        right = np.concatenate([x[:, 1:], x[:, -1:]], 1)
        o = np.empty((x.shape[0], 2 * x.shape[1]))
        o[:, 0::2], o[:, 1::2] = 0.25 * left + 0.75 * x, 0.75 * x + 0.25 * right
        x = o
    if vs:
        up = np.concatenate([x[:1], x[:-1]], 0)
        down = np.concatenate([x[1:], x[-1:]], 0)
        o = np.empty((2 * x.shape[0], x.shape[1]))
        o[0::2], o[1::2] = 0.75 * x + 0.25 * up, 0.25 * down + 0.75 * x
        x = o
    return x[:h, :w]


def ycbcr_model(coded, maxval, w, h, shifts, y_offset=128 / 255):
    """Cb, Y, Cr integer planes -> RGB in float64 (jxl-color/src/ycbcr.rs with the f32 constants)."""
    cb, y, cr = (jpeg_upsample(c.astype(np.float64) / maxval, hs, vs, w, h) for c, (hs, vs) in zip(coded, shifts))
    f32 = lambda v: float(np.float32(v))  # noqa: E731
    y = y + y_offset
    return np.stack([y + f32(1.402) * cr,
                     y + f32(np.float32(-0.114) * np.float32(1.772) / np.float32(0.587)) * cb +
                     f32(np.float32(-0.299) * np.float32(1.402) / np.float32(0.587)) * cr,
                     y + f32(1.772) * cb])


def chain_model(x, total, order=None):
    """features::upsample: floor(total / 3) passes of 8x, then one of 2x or 4x, each pass on the previous one's whole
    output. Returns (out, bound) with the bound of each pass carried through the next one's kernel."""
    factors = order or [8] * (total // 3) + {0: [], 1: [2], 2: [4]}[total % 3]
    bound = np.zeros_like(x, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    for k in factors:
        prev = np.kron(bound, np.ones((k, k)))
        x, b = fm.upsample(x, k)
        gain = np.abs(fm._weights(fm.UP_WEIGHTS[k])).sum()  # bounds the sum of |kernel| of every phase
        bound = b + gain * prev
    return x, bound


SHIFTS = {"444": [(0, 0)] * 3, "420": [(1, 1), (0, 0), (1, 1)], "422": [(1, 0), (0, 0), (1, 0)], "440": [(0, 1), (0, 0), (0, 1)]}


# ---- tests ----

@pytest.mark.parametrize("args,extra,size,sha", DIGESTS)
def test_default_encoder_output_unchanged(args, extra, size, sha):
    data = bench.synth_frame(*args, extra=extra)
    assert len(data) == size
    assert hashlib.sha256(data).hexdigest() == sha


@pytest.mark.parametrize("mode,w,h", YCBCR)
def test_ycbcr_modular(oracle, tmp_path, mode, w, h):
    data, raw = encode(tmp_path, w, h, ["--ycbcr", mode])
    img = oracle.OracleImage(data, threads=4, capture=True)
    coded, same = coded_equal(img, raw)
    assert same, "the oracle's coded channels differ from the encoder's samples"
    for c, (hs, vs) in zip(coded, SHIFTS[mode]):  # shift_size: ceil(n / 2), or twice that for a full-size channel
        assert c.shape == (((h + 1) // 2 * (2 - vs)) if any(s[1] for s in SHIFTS[mode]) else h,
                           ((w + 1) // 2 * (2 - hs)) if any(s[0] for s in SHIFTS[mode]) else w)
    up = img.stage("jpeg_upsampled")
    assert [p.shape for p in up] == [(h, w)] * 3
    got = img.frame(0)[0]
    assert got.shape == (3, h, w)
    want = ycbcr_model(coded, 255, w, h, SHIFTS[mode])
    err = np.abs(got.astype(np.float64) - want)
    assert err.max() <= 4e-6, f"max error {err.max()}"
    # the model must be able to fail: Y without its 128/255 offset
    assert np.abs(got - ycbcr_model(coded, 255, w, h, SHIFTS[mode], y_offset=0)).max() > 0.4


def check_extras(img, raw, up, extras, w, h, ncol_coded):
    coded, same = coded_equal(img, raw)
    assert same, "the oracle's coded channels differ from the encoder's samples"
    got, ncol, _ = img.frame(0)
    assert ncol == 3 and got.shape == (3 + len(extras), h, w)
    ushift = int(np.log2(up))
    for i, e in enumerate(extras):
        _, bits, dim_shift, ec_up = e.split(":")
        total = int(np.log2(int(ec_up))) + int(dim_shift)
        c = coded[ncol_coded + i]
        s = total - ushift
        cw, ch = -(-w // up), -(-h // up)
        assert c.shape == (-(-ch // (1 << s)), -(-cw // (1 << s)))
        x = c.astype(np.float64) / ((1 << int(bits)) - 1)
        plane = got[3 + i].astype(np.float64)
        if total == 0:
            assert np.array_equal(plane, x.astype(np.float32))
            continue
        want, bound = chain_model(x, total)
        want, bound = want[:h, :w], bound[:h, :w]
        assert (np.abs(plane - want) <= bound + 1e-6).all(), f"channel {i}: max error {np.abs(plane - want).max()}"
        if total >= 4:  # a planted model error (the chain in another order) must fail
            wrong, _ = chain_model(x, total, order={4: [2, 8], 5: [4, 8], 6: [4, 4, 4]}[total])
            assert np.abs(plane - wrong[:h, :w]).max() > 1e-4
    assert len(img.stage("extra_upsampled")) == len(extras)
    return got


@pytest.mark.parametrize("up,extras,w,h", EXTRA)
def test_extra_channels_at_own_resolution(oracle, tmp_path, up, extras, w, h):
    data, raw = encode(tmp_path, w, h, extra_args(up, extras))
    check_extras(oracle.OracleImage(data, threads=8, capture=True), raw, up, extras, w, h, 3)


@pytest.mark.parametrize("extras,w,h", EXTRA_VARDCT)
def test_extra_channels_in_vardct_frames(oracle, tmp_path, extras, w, h):
    data, raw = encode(tmp_path, w, h, extra_args(1, extras), modular=False)
    got = check_extras(oracle.OracleImage(data, threads=8, capture=True), raw, 1, extras, w, h, 0)
    # the colour channels are those of the same frame without extra channels
    plain, _ = encode(tmp_path, w, h, [], modular=False)
    want = oracle.OracleImage(plain, threads=8).frame(0)[0]
    assert np.array_equal(got[:3].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("total", [4, 5, 6])
def test_chain_each_pass_from_the_previous_one(oracle, tmp_path, total):
    """Each pass of a chained factor against the model applied to the oracle's output of the pass before it. A VarDCT
    frame draws its extra channels apart from its colour content, so a second frame sized to code the same samples at
    shift 3 gives the first 8x pass exactly as the chain computes it."""
    w, h = 1100, 700
    dim_shift, ec_up = {4: (1, 8), 5: (2, 8), 6: (3, 8)}[total]
    data, raw = encode(tmp_path, w, h, extra_args(1, [f"alpha:8:{dim_shift}:{ec_up}"]), modular=False)
    cw, ch = -(-w // (1 << total)), -(-h // (1 << total))
    first, raw8 = encode(tmp_path, cw * 8, ch * 8, extra_args(1, ["alpha:8:3:1"]), modular=False)
    assert np.array_equal(raw, raw8)
    x = raw.reshape(ch, cw).astype(np.float64) / 255
    mid = oracle.OracleImage(first, threads=8).frame(0)[0][3]
    want, bound = fm.upsample(x, 8)
    assert (np.abs(mid - want) <= bound + 1e-6).all()
    plane = oracle.OracleImage(data, threads=8).frame(0)[0][3]
    want, bound = fm.upsample(mid, {4: 2, 5: 4, 6: 8}[total])
    assert (np.abs(plane - want[:h, :w]) <= bound[:h, :w] + 1e-6).all()


@pytest.mark.parametrize("mode", ["420", "422"])
def test_ycbcr_modular_filters_sit_between_chroma_upsampling_and_colour(oracle, tmp_path, mode):
    """Render order: chroma upsampling, then Gaborish and EPF (sigma_for_modular) on Cb, Y, Cr, then YCbCr -> RGB."""
    w, h = 301, 157
    data, raw = encode(tmp_path, w, h, ["--ycbcr", mode, "--modular-filters", "1.5"])
    img = oracle.OracleImage(data, threads=4, capture=True)
    coded, same = coded_equal(img, raw)
    assert same
    up = np.stack(img.stage("jpeg_upsampled")).astype(np.float64)
    want = np.stack([jpeg_upsample(c.astype(np.float64) / 255, hs, vs, w, h) for c, (hs, vs) in zip(coded, SHIFTS[mode])])
    assert np.abs(up - want).max() <= 1e-6
    filtered = np.stack(img.stage("epf")).astype(np.float64)
    assert np.abs(filtered - up).max() > 1e-3, "the filters left the planes as they were"
    got = img.frame(0)[0]
    identity = [(0, 0)] * 3  # the filtered planes are at full size already
    assert np.abs(got - ycbcr_model(filtered * 255, 255, w, h, identity)).max() <= 4e-6
    assert np.abs(got - ycbcr_model(up * 255, 255, w, h, identity)).max() > 1e-3


@pytest.mark.parametrize("case", ["ycbcr420", "extras", "vardct_extras"])
def test_host_emulation_matches_oracle(oracle, tmp_path, case):
    args = {"ycbcr420": ["--ycbcr", "420"], "extras": extra_args(2, ["alpha:8:1:2", "unknown:12:3:8"]),
            "vardct_extras": extra_args(1, ["alpha:8:1:1", "unknown:12:3:8"])}[case]
    data, _ = encode(tmp_path, 2100, 301, args, modular=case != "vardct_extras")
    want = oracle.OracleImage(data, threads=8).frame(0)[0]
    got = oracle.OracleImage(data, threads=8, emu=True).frame(0)[0]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_ec_upsampling_below_colour_upsampling_is_a_bitstream_error(oracle, tmp_path):
    data, _ = encode(tmp_path, 130, 70, extra_args(4, ["alpha:8:0:2"]))
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(data)
    assert e.value.code == 1  # JXLB_ERR_BITSTREAM


# What the reference's fuzz findings that used to stop at the removed checks do now
FUZZ = {"ec_upsampling": 1, "invalid_alpha_ref": 1, "noise_on_invisible_frame": 1, "modular_jpeg_upsampling": 1,
        "modular_jpeg_upsampling_2": 1, "patchref_idx": 1, "upsample_separate_ec": 2, "upsampling_sum_not_finite": 3}
REMOVED = ("YCbCr modular frames are outside", "chroma-subsampled Modular frames are not implemented",
           "extra-channel upsampling differs from colour", "dim_shift extra channels not supported")


@pytest.mark.parametrize("name", sorted(FUZZ))
def test_fuzz_findings_pass_the_removed_checks(oracle, name):
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(fixture_bytes("fuzz_findings", name + ".fuzz"))
    assert not any(m in str(e.value) for m in REMOVED)
    assert e.value.code == FUZZ[name]
    if name == "upsample_separate_ec":  # patches with an extra channel upsampled apart from the colour channels
        assert "patches on a frame whose extra channel" in str(e.value)
