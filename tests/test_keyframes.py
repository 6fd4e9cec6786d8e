"""Keyframe index and segments (host/frame_index.cc) on the CPU: the counts jxlb_image_keyframes gives, the segment
boundaries of synthetic animations, and every keyframe decoded from its own segment on the oracle against the oracle's
full sequential decode, bit for bit. That equality is what proves the dependency rule and the noise seed counts."""
import glob
import os

import numpy as np
import pytest

import jxl_oxide_b200 as J
import keyframe_lib as K
import oracle_lib


def _full(data):
    o = oracle_lib.OracleImage(data, threads=4)
    return o, [o.frame(i)[0] for i in range(o.num_frames)]


@pytest.mark.parametrize("name", K.FIXTURES)
def test_keyframe_count_matches_oracle(name):
    data = K.fixture(name)
    try:
        o = oracle_lib.OracleImage(data, threads=4)
    except oracle_lib.OracleError:
        pytest.skip("the oracle refuses this stream")
    nk, ns, st = J.image_keyframes(data)
    assert st == J.OK
    assert nk == o.num_frames
    assert 1 <= ns <= nk
    if name not in K.ANIMATIONS:
        assert nk == 1


def test_issue_24_has_nine_keyframes():
    assert J.image_keyframes(K.fixture("issue_24"))[0] == 9


@pytest.mark.parametrize("frames", [1, 2, 7])
def test_synthetic_segment_counts(frames):
    assert J.image_keyframes(K.animation("independent", frames)) == (frames, frames, J.OK)
    assert J.image_keyframes(K.animation("chain", frames)) == (frames, 1, J.OK)


def test_mixed_segment_boundaries():
    # frames 0..7: frames 0, 3 and 6 replace the whole canvas; the others replace a sub-rectangle of slot 1 and save to
    # slot 1, except the last frame of each chain (2, 5), which saves to slot 2 that no frame reads; frame 1 has
    # duration 0, so it is composed into keyframe 1 (frame 2). Keyframes: frames 0, 2, 3, 4, 5, 6, 7 -> 0..6.
    data = K.animation("mixed", 8)
    assert J.image_keyframes(data) == (7, 3, J.OK)
    segs, err = K.segments(data)
    assert err == 0
    assert segs == [(0, 2), (2, 3), (5, 2)]


@pytest.mark.parametrize("name", K.ANIMATIONS + ["opsin_inverse", "noise", "patches", "bike", "blendmodes"])
def test_fixture_keyframes_from_segments_equal_full_decode(name):
    data = K.fixture(name)
    _, frames = _full(data)
    for k, want in enumerate(frames):
        got = K.decode_keyframe(data, k)
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"keyframe {k} differs"


@pytest.mark.parametrize("mode", K.MODES)
def test_synthetic_keyframes_from_segments_equal_full_decode(mode):
    data = K.animation(mode, 7)
    o, frames = _full(data)
    assert len(frames) == J.image_keyframes(data)[0]
    for k, want in enumerate(frames):
        got = K.decode_keyframe(data, k)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{mode}: keyframe {k} differs"


def test_synthetic_frames_are_the_encoded_frames():
    # an independent frame is the single-frame stream of its seed; a chained one is the previous canvas with the
    # sub-rectangle replaced by its own single-frame stream
    import bench
    w, h = 300, 200
    ind = _full(K.animation("independent", 3, w, h, seed=5))[1]
    for i, f in enumerate(ind):
        alone = oracle_lib.OracleImage(bench.synth_frame(w, h, 5 + i), threads=4).frame(0)[0]
        assert np.array_equal(f.view(np.uint32), alone.view(np.uint32))
    chain = _full(K.animation("chain", 3, w, h, seed=5))[1]
    x0, y0, cw, ch = K.synth_anim.frame_plan("chain", 3, w, h)[1][0]
    for i in (1, 2):
        sub = oracle_lib.OracleImage(bench.synth_frame(cw, ch, 5 + i), threads=4).frame(0)[0]
        want = chain[i - 1].copy()
        want[:, y0:y0 + ch, x0:x0 + cw] = sub
        assert np.array_equal(chain[i].view(np.uint32), want.view(np.uint32))


def test_truncated_animation_keeps_earlier_segments():
    data = K.animation("independent", 5)
    cut = data[: len(data) - 200]  # inside the last frame's sections
    nk, ns, st = J.image_keyframes(cut)
    assert (nk, ns) == (5, 5) and st == J.ERR_EOF
    segs, err = K.segments(cut)
    assert err == J.ERR_EOF and segs[-1] == (4, 1)
    _, frames = _full(data)
    for k in range(4):
        assert np.array_equal(K.decode_keyframe(cut, k).view(np.uint32), frames[k].view(np.uint32))
    with pytest.raises(oracle_lib.OracleError) as e:
        K.decode_keyframe(cut, 4)
    assert e.value.code == J.ERR_EOF


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(K.GOLDEN, "fuzz_findings", "*.fuzz"))),
                         ids=lambda p: os.path.basename(p))
def test_fuzz_findings_index_without_crashing(path):
    with open(path, "rb") as f:
        data = f.read()
    try:
        nk, ns, st = J.image_keyframes(data)
    except J.JxlError:
        return
    assert nk >= ns and (ns >= 1 or nk == 0)
    for k in range(min(nk, 3)):
        try:
            K.decode_keyframe(data, k)
        except oracle_lib.OracleError:
            pass


def test_image_keyframes_rejects_garbage():
    with pytest.raises(J.JxlError):
        J.image_keyframes(b"\x00\x01\x02")
