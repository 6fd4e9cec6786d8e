"""Channels coded below the frame's resolution on the device: YCbCr Modular frames with chroma subsampling and extra
channels with dim_shift or their own upsampling, in Modular and VarDCT frames, decode bit for bit like the oracle,
through jxlb_decode (final planes and stages) and through the frame pipeline (host and device outputs, packed alpha)."""
import ctypes

import numpy as np
import pytest

from test_channel_shifts import encode, extra_args

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200, method="thread")]

KINDS = [(["--ycbcr", m], w, h, True) for m in ("444", "420", "422", "440") for (w, h) in [(257, 129), (5, 1), (1, 7), (513, 270)]]
KINDS += [(extra_args(up, ex), w, h, True) for (up, ex, w, h) in [
    (1, ["alpha:8:2:1", "spot:12:0:1"], 600, 300),
    (1, ["alpha:8:0:8", "unknown:8:3:8"], 2100, 333),
    (2, ["alpha:8:0:4", "spot:12:1:2"], 517, 301),
    (2, ["unknown:16:2:8"], 4200, 260),
    (4, ["alpha:8:2:4", "unknown:1:0:8"], 1030, 77),
    (8, ["alpha:8:3:8", "spot:10:0:8"], 4100, 37),
    (2, ["alpha:8:1:2"], 9, 1),
]]
KINDS += [(["--ycbcr", "420", "--upsampling", "2", "--extra", "alpha:8:1:4"], 700, 501, True),
          (["--ycbcr", "422", "--modular-filters", "1.5"], 301, 157, True)]
KINDS += [(extra_args(1, ex), w, h, False) for (ex, w, h) in [
    (["alpha:8:2:1"], 600, 300),
    (["alpha:8:1:1", "unknown:12:3:8", "spot:10:0:2"], 2100, 900),
    (["alpha:8:0:4", "unknown:16:2:8"], 4200, 260),
    (["alpha:8:3:8"], 2600, 700),
    (["alpha:8:1:1"], 1, 1),
    (["spot:8:0:8", "alpha:8:1:2"], 257, 9),
]]
IDS = [("modular " if m else "vardct ") + " ".join(a) + f" {w}x{h}" for a, w, h, m in KINDS]
STAGES = ["jpeg_upsampled", "upsampled", "extra_upsampled", "pre_filter", "gaborish", "epf", "rgb"]


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("args,w,h,modular", KINDS, ids=IDS)
def test_decode_matches_oracle(dec, oracle, tmp_path, args, w, h, modular):
    data, _ = encode(tmp_path, w, h, args, modular=modular)
    dec.set_capture(True)
    dec.set_fuse_filters(False)  # every filter stage on its own, to compare it
    try:
        dec.decode(data)
        got = dec.frame_planar(0)
        img = oracle.OracleImage(data, threads=8, capture=True)
        want = img.frame(0)[0]
        assert got.shape == want.shape
        assert np.array_equal(_bits(got), _bits(want))
        for st in STAGES:
            gs, ws = dec.stage(st), img.stage(st)
            assert len(gs) == len(ws), st
            for g, wv in zip(gs, ws):
                assert np.array_equal(_bits(g), _bits(wv)), st
        assert np.array_equal(dec.frame_to_buffer(0, np.uint8), img.frame_to_buffer(0, np.uint8))
        assert np.array_equal(dec.frame_to_buffer(0, np.uint16), img.frame_to_buffer(0, np.uint16))
    finally:
        dec.set_capture(False)
        dec.set_fuse_filters(True)
    if not modular:  # production path: filters and colour fused
        dec.decode(data)
        assert np.array_equal(_bits(dec.frame_planar(0)), _bits(want))


def test_pipeline_outputs_match_oracle(oracle, tmp_path):
    import torch
    import jxl_oxide_b200 as J
    cases = [k for k in KINDS if k[1] * k[2] > 100]
    datas, planar, packed = [], [], []
    for i, (args, w, h, modular) in enumerate(cases):
        d, _ = encode(tmp_path, w, h, args, seed=i + 3, modular=modular)
        img = oracle.OracleImage(d, threads=8)
        datas.append(d)
        planar.append(img.frame(0)[0])
        packed.append(img.frame_to_buffer(0, np.uint8))  # RGBA where the frame has alpha at reduced resolution
        img.close()
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for i, d in enumerate(datas):
            p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=i)
            p.submit(data=d, mode=p.OUT_U8, tag=100 + i)
            p.preload(i, d)
        dev = [torch.zeros(w.shape, dtype=torch.uint8, device="cuda:0") for w in packed]
        for i in range(len(datas)):
            p.submit(slot=i, out=dev[i], tag=200 + i)
        seen = set()
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            kind, i = divmod(tag, 100)
            if kind == 2:
                seen.add(tag)
                continue
            want = planar[i] if kind == 0 else packed[i]
            assert nbytes == want.nbytes, tag
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=want.dtype).reshape(want.shape).copy()
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), tag
            seen.add(tag)
        torch.cuda.synchronize()
        for i in range(len(datas)):
            assert np.array_equal(dev[i].cpu().numpy(), packed[i]), f"device output {i}"
        assert len(seen) == 3 * len(datas)
    finally:
        p.close()


def test_large_frame_with_reduced_alpha_at_bench_defaults(oracle, tmp_path):
    """A 7680x4320 VarDCT frame with 8-bit alpha at dim_shift 2 through a pipeline with the bench's 64 workers and 16
    heavy slots decodes like the oracle (what does not fit a heavy slot's slab is taken from the memory pool, so this
    shows the result at bench scale, not the slab size)."""
    import jxl_oxide_b200 as J
    data, _ = encode(tmp_path, 7680, 4320, extra_args(1, ["alpha:8:2:1"]), modular=False)
    want = oracle.OracleImage(data, threads=16).frame(0)[0]
    p = J.Pipeline(0, workers=64, heavy_frames=16)
    try:
        for i in range(3):
            p.submit(data=data, mode=p.OUT_PLANAR_F32, tag=i)
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            assert nbytes == want.nbytes
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), dtype=np.float32).reshape(want.shape).copy()
            p.release_output(addr)
            assert np.array_equal(_bits(got), _bits(want)), tag
    finally:
        p.close()


def _least_budget(J, data, hi=1 << 28, step=1 << 16):
    """The smallest jxlb_decoder_create_ex budget (to `step` bytes) under which `data` decodes, and the error one step
    below it."""
    lo, err = 0, None
    while hi - lo > step:
        mid = (lo + hi) // 2 // step * step
        d = J.Decoder(0, mem_limit=mid)
        try:
            d.decode(data)
            hi = mid
        except J.JxlError as e:
            lo, err = mid, e
        finally:
            d.close()
    return hi, err


def test_memory_limit_counts_the_upsampled_extra_channels(tmp_path):
    """The same VarDCT frame with and without six extra channels coded at 1/8 resolution. Without them the budget peaks
    in the filter stage (three coefficient planes and three output planes); after it the frame holds three colour planes,
    so six full-size extra planes take it at least three planes past that peak. The least budget must grow by at least
    two planes, and a budget just below it fails cleanly with JXLB_ERR_OUT_OF_MEMORY."""
    import jxl_oxide_b200 as J
    w, h = 1024, 1024
    plain, _ = encode(tmp_path, w, h, [], modular=False)
    with_ec, _ = encode(tmp_path, w, h, extra_args(1, ["alpha:8:3:1"] + ["unknown:8:3:1"] * 5), modular=False)
    base, _ = _least_budget(J, plain)
    need, err = _least_budget(J, with_ec)
    assert need - base >= 2 * w * h * 4, (base, need)
    assert err is not None and err.code == J.ERR_OUT_OF_MEMORY
    d = J.Decoder(0, mem_limit=need)  # the decoder is usable at the budget that fits
    try:
        d.decode(with_ec)
        assert d.frame_planar(0).shape == (9, h, w)
    finally:
        d.close()
