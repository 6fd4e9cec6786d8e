"""Frames saved before the colour transform, reference-only frames saved after it (also upsampled), blending onto a
slot saved before it, and previews, on the oracle. Each check compares with frames decoded on their own as plain shown
frames, so none of them rests on the composition code it checks."""
import numpy as np
import pytest

import frame_kinds_lib as F
import jxl_oxide_b200 as J
import keyframe_lib as K
import oracle_lib


def _frames(data, output_colour=0):
    o = oracle_lib.OracleImage(data, output_colour=output_colour, threads=4)
    return [o.frame(k)[0] for k in range(o.num_frames)]


def _bits(a):
    return a.view(np.uint32)


def _outside(a, sub=F.SUB):
    x0, y0, w, h = sub
    m = np.ones(a.shape[-2:], dtype=bool)
    m[y0:y0 + h, x0:x0 + w] = False
    return a[:, m]


@pytest.mark.parametrize("output_colour", [0, 1, 2])
def test_replace_frames_saved_before_the_transform_equal_those_saved_after(output_colour):
    # a full-canvas Replace copies the frame as it is: the transform commutes with it
    before, after = _frames(F.replace_chain(True), output_colour), _frames(F.replace_chain(False), output_colour)
    assert len(before) == len(after) == 3
    for a, b in zip(before, after):
        assert np.array_equal(_bits(a), _bits(b))


@pytest.mark.parametrize("output_colour", [0, 1])
def test_add_onto_a_slot_saved_before_the_transform(output_colour):
    # the base is taken from the slot as it is (XYB) and not converted; the added frame was converted before it was
    # composed, and the canvas keeps the added frame's state, so nothing converts the base afterwards
    base_xyb = _frames(F.shown_alone(), 2)[0]
    x0, y0, w, h = F.SUB
    top = _frames(K.synth_anim.synth_frames(w, h, [dict()], F.SEED + 1), output_colour)[0]
    want = base_xyb.copy()
    want[:, y0:y0 + h, x0:x0 + w] = base_xyb[:, y0:y0 + h, x0:x0 + w] + top
    got = _frames(F.add_onto_slot(True), output_colour)[0]
    assert np.array_equal(_bits(got), _bits(want))
    # the same stream with the base saved after the transform: the base is in the output encoding
    after = _frames(F.add_onto_slot(False), output_colour)[0]
    base = _frames(F.shown_alone(), output_colour)[0]
    assert np.array_equal(_bits(_outside(after)), _bits(_outside(base)))


@pytest.mark.parametrize("upsampling", [1, 2])
@pytest.mark.parametrize("output_colour", [0, 1, 2])
def test_reference_frame_saved_after_the_transform_records_the_signalled_encoding(upsampling, output_colour):
    # whatever output is asked for, the slot holds the frame in the image's signalled encoding (sRGB): the frame as it
    # is shown on its own with output_colour 0
    got = _frames(F.reference_then_crop(upsampling), output_colour)[0]
    shown = _frames(F.shown_alone(upsampling), 0)[0]
    assert np.array_equal(_bits(_outside(got)), _bits(_outside(shown)))


def test_upsampled_reference_frame_saved_before_the_transform_stays_in_xyb():
    got = _frames(F.reference_then_crop(2, save_before_ct=True), 0)[0]
    shown = _frames(F.shown_alone(2), 2)[0]
    assert np.array_equal(_bits(_outside(got)), _bits(_outside(shown)))


@pytest.mark.parametrize("default_header", [False, True], ids=["cropped_header", "default_header"])
def test_preview_is_skipped(default_header):
    # with an all-default header the preview frame has the image's size, not the declared 64 x 48: its TOC has the
    # image's group count, and reading it with the preview's would land inside the preview's sections
    still, with_preview = F.noise_still(), F.noise_with_preview(default_header)
    assert len(with_preview) > len(still)
    assert J.image_keyframes(with_preview) == J.image_keyframes(still) == (1, 1, J.OK)
    want = _frames(still)
    got = _frames(with_preview)
    assert len(got) == len(want) == 1
    # the noise seed counts the frames before this one: the preview is not among them
    assert np.array_equal(_bits(got[0]), _bits(want[0]))
    assert np.array_equal(_bits(K.decode_keyframe(with_preview, 0)), _bits(want[0]))


def test_truncated_preview_fails_with_eof():
    data = F.noise_with_preview()
    head = len(K.synth_anim.image_header(F.W, F.H, False, preview=F.PREVIEW).bytes())
    for cut in (head + 3, head + 40):
        with pytest.raises(oracle_lib.OracleError) as e:
            oracle_lib.OracleImage(data[:cut], threads=2)
        assert e.value.code == J.ERR_EOF
        with pytest.raises(J.JxlError) as e:
            J.image_keyframes(data[:cut])
        assert e.value.code == J.ERR_EOF


def test_icc_image_header_is_reused_as_is():
    alone = F.icc_image([dict()])
    o = oracle_lib.OracleImage(alone, output_colour=2, threads=2)
    assert (o.width, o.height, o.num_frames) == (F.ICC_SIZE, F.ICC_SIZE, 1)
    assert o.original_icc() == oracle_lib.OracleImage(K.fixture("grayscale"), threads=2).original_icc() != b""


@pytest.mark.parametrize("base", [dict(reference=True, save_as=1), dict(reference=True, save_as=1, save_before_ct=True),
                                  dict(save_as=1, save_before_ct=True)], ids=["reference_after_ct",
                                                                             "reference_before_ct", "regular_before_ct"])
def test_icc_blend_onto_a_slot_before_the_transform(base):
    # under an ICC profile the reference records every frame in XYB and converts the composed canvas at the end; the
    # planner converts the cropped frame before composing it, so composing it onto an XYB slot is refused
    data = F.icc_image([base, dict(crop=F.ICC_SUB, source=1)])
    for output_colour in (0, 1):
        with pytest.raises(oracle_lib.OracleError) as e:
            _frames(data, output_colour)
        assert e.value.code == J.ERR_UNSUPPORTED
    # with XYB output nothing is converted: the canvas outside the crop is the first frame as coded
    got = _frames(data, 2)[0]
    alone = _frames(F.icc_image([dict()]), 2)[0]
    assert np.array_equal(_bits(_outside(got, F.ICC_SUB)), _bits(_outside(alone, F.ICC_SUB)))


@pytest.mark.parametrize("name", sorted(F.STREAMS))
def test_keyframes_from_segments_equal_full_decode(name):
    data = F.STREAMS[name]
    frames = _frames(data)
    assert J.image_keyframes(data)[0] == len(frames)
    for k, want in enumerate(frames):
        assert np.array_equal(_bits(K.decode_keyframe(data, k)), _bits(want))
