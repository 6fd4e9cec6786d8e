"""GPU tests of keyframes one at a time: jxlb_decode_keyframe against keyframe k of jxlb_decode, bit for bit, its memory
bound under an allocation budget, and jxlb_pipeline_submit_keyframes in every out mode against the oracle, with caller
buffers and with the pipeline's ring, interleaved with single-frame images, and with a truncated animation."""
import ctypes

import numpy as np
import pytest

import jxl_oxide_b200 as J
import keyframe_lib as K
import oracle_lib

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

SYNTH = {mode: K.animation(mode, 7) for mode in K.MODES}


def _inputs():
    return [(n, K.fixture(n)) for n in K.ANIMATIONS + ["opsin_inverse", "noise", "patches"]] + \
           [(f"synth_{m}", d) for m, d in SYNTH.items()]


@pytest.mark.parametrize("name,data", _inputs(), ids=[n for n, _ in _inputs()])
def test_decode_keyframe_equals_full_decode(name, data):
    full, one = J.Decoder(0), J.Decoder(0)
    full.decode(data)
    n = full.num_frames()
    assert n == J.image_keyframes(data)[0]
    for k in range(n):
        one.decode_keyframe(data, k)
        assert one.num_frames() == 1
        a, b = full.frame_planar(k), one.frame_planar(0)
        assert a.shape == b.shape
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{name}: keyframe {k} differs"
        assert np.array_equal(full.frame_to_buffer(k), one.frame_to_buffer(0))
    full.close()
    one.close()


def test_decode_keyframe_fits_a_budget_the_full_decode_exceeds():
    data = K.fixture("animation_icos4d")
    nk = J.image_keyframes(data)[0]
    budget = None
    for mib in (4, 8, 16, 24, 32, 48, 64, 96, 128, 192, 256):
        d = J.Decoder(0, mem_limit=mib << 20)
        try:
            d.decode_keyframe(data, nk - 1)
            budget = mib << 20
            break
        except J.JxlError as e:
            assert e.code == J.ERR_OUT_OF_MEMORY
        finally:
            d.close()
    assert budget is not None
    d = J.Decoder(0, mem_limit=budget)
    with pytest.raises(J.JxlError) as e:
        d.decode(data)
    assert e.value.code == J.ERR_OUT_OF_MEMORY
    d.decode_keyframe(data, nk - 1)
    ref = J.Decoder(0)
    ref.decode(data)
    assert np.array_equal(d.frame_planar(0).view(np.uint32), ref.frame_planar(nk - 1).view(np.uint32))
    d.close()
    ref.close()


def _want(data, mode):
    o = oracle_lib.OracleImage(data, threads=16)
    if mode == 1:
        return [o.frame(k)[0] for k in range(o.num_frames)]
    dt = np.uint8 if mode in (2, 4) else np.uint16
    return [o.frame_to_buffer(k, dt) for k in range(o.num_frames)]


def _as_array(addr, nbytes, dtype, shape):
    buf = (ctypes.c_uint8 * nbytes).from_address(addr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()


def _submit_all(pipe, items, mode, use_ring, device_out):
    """Submits every item as keyframes; returns {tag: (data, wants, out array or None)}."""
    import torch
    jobs = {}
    for name, data, slot in items:
        wants = _want(data, mode)
        out = None
        if not use_ring:
            shape = (len(wants),) + wants[0].shape
            if device_out:
                out = torch.empty(shape, dtype=torch.uint8 if mode == 4 else torch.int16, device="cuda:0")
            else:
                out = np.zeros(shape, dtype=wants[0].dtype)
        tag = pipe.submit_keyframes(None if slot is not None else data, slot=-1 if slot is None else slot, out=out, mode=mode)
        jobs[tag] = (name, wants, out)
    return jobs


def _collect(pipe, jobs, mode, use_ring):
    seen = {tag: [] for tag in jobs}
    while pipe.in_flight:
        tag, k, addr, nbytes = pipe.wait_keyframe(want_output=True)
        name, wants, out = jobs[tag]
        want = wants[k]
        if use_ring:
            got = _as_array(addr, nbytes, want.dtype, want.shape)
            pipe.release_output(addr)  # consumed: back to the ring at once
        elif hasattr(out, "data_ptr"):
            got = out[k].cpu().numpy().view(want.dtype)
        else:
            got = out[k]
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), f"{name}: keyframe {k} differs"
        seen[tag].append(k)
    for tag, (name, wants, _) in jobs.items():
        assert sorted(seen[tag]) == list(range(len(wants))), name


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("use_ring", [False, True], ids=["caller", "ring"])
def test_pipeline_keyframes_every_mode(mode, use_ring):
    if mode >= 4 and use_ring:
        pytest.skip("device out modes always write the caller's buffer")
    pipe = J.Pipeline(0, workers=3, heavy_frames=2)
    items = [("independent", SYNTH["independent"], None), ("opsin_inverse", K.fixture("opsin_inverse"), None),
             ("chain", SYNTH["chain"], None), ("mixed", SYNTH["mixed"], None),
             ("animation_newtons_cradle", K.fixture("animation_newtons_cradle"), None), ("noise", K.fixture("noise"), None)]
    pipe.preload(3, SYNTH["mixed"])
    items.append(("mixed_slot", SYNTH["mixed"], 3))
    jobs = _submit_all(pipe, items, mode, use_ring, mode >= 4)
    _collect(pipe, jobs, mode, use_ring)
    pipe.close()


def test_pipeline_segment_longer_than_the_ring():
    # the ring has 6 buffers: a chained animation of 16 keyframes is one segment whose worker must wait for buffers
    pipe = J.Pipeline(0, workers=2, heavy_frames=2)
    data = K.animation("chain", 16)
    jobs = _submit_all(pipe, [("chain16", data, None), ("independent", SYNTH["independent"], None)], 2, True, False)
    _collect(pipe, jobs, 2, True)
    pipe.close()


def test_pipeline_keyframes_and_plain_frames_together():
    pipe = J.Pipeline(0, workers=2, heavy_frames=2)
    data = SYNTH["independent"]
    plain = K.fixture("opsin_inverse")
    t_plain = pipe.submit(plain)
    t_kf = pipe.submit_keyframes(data)
    got = {}
    while pipe.in_flight:
        tag, k = pipe.wait_keyframe()
        got.setdefault(tag, []).append(k)
    assert got[t_plain] == [-1]
    assert sorted(got[t_kf]) == list(range(7))
    # jxlb_pipeline_wait reports keyframes too: one report per keyframe
    pipe.submit_keyframes(data)
    n = 0
    while pipe.in_flight:
        pipe.wait()
        n += 1
    assert n == 7
    pipe.close()


def test_truncated_animation_fails_only_its_last_segment():
    data = K.animation("independent", 5)
    cut = data[: len(data) - 200]
    wants = _want(data, 2)
    pipe = J.Pipeline(0, workers=3, heavy_frames=2)
    pipe.submit_keyframes(cut, mode=2)
    ok, failed = [], []
    while pipe.in_flight:
        try:
            tag, k, addr, nbytes = pipe.wait_keyframe(want_output=True)
            got = _as_array(addr, nbytes, np.uint8, wants[k].shape)
            pipe.release_output(addr)
            assert np.array_equal(got, wants[k])
            ok.append(k)
        except J.JxlError as e:
            assert e.code == J.ERR_EOF
            failed.append(e.keyframe)
    assert sorted(ok) == [0, 1, 2, 3] and failed == [4]
    # a chain cut short: the keyframes before the cut are delivered, the rest of the segment reports the error
    chain = K.animation("chain", 5)
    pipe.submit_keyframes(chain[: len(chain) - 100], mode=2)
    ok, failed = [], []
    while pipe.in_flight:
        try:
            tag, k, addr, nbytes = pipe.wait_keyframe(want_output=True)
            pipe.release_output(addr)
            ok.append(k)
        except J.JxlError as e:
            failed.append(e.keyframe)
    assert sorted(ok) == [0, 1, 2, 3] and failed == [4]
    pipe.close()
