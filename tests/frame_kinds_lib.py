"""Synthetic streams of the frame kinds whose colour state differs from a plain shown frame's (tools/synth_anim.py):
frames saved before the colour transform, reference-only frames saved after it (also upsampled), blending onto a slot
saved before it, and still images with a preview frame in front. Test infrastructure only."""
import os

import bench
import keyframe_lib as K

W, H = 300, 200
SUB = (60, 40, 150, 100)  # x0, y0, width, height of the cropped frames
SEED = 11
synth_anim = K.synth_anim


def replace_chain(save_before_ct):
    """Three full-canvas Replace keyframes saved to slot 1 (which signals save_before_ct), the last one not saved."""
    return synth_anim.synth_frames(W, H, [dict(save_as=1, save_before_ct=save_before_ct)] * 2 + [dict()], SEED)


def add_onto_slot(save_before_ct):
    """A hidden full-canvas frame saved to slot 1, then the last frame, cropped, added onto slot 1."""
    return synth_anim.synth_frames(W, H, [dict(duration=0, save_as=1, save_before_ct=save_before_ct),
                                          dict(crop=SUB, source=1, add=True)], SEED)


def reference_then_crop(upsampling=1, save_before_ct=False):
    """A reference-only frame saved to slot 1, read back through the last frame: a cropped Replace onto slot 1."""
    return synth_anim.synth_frames(W, H, [dict(reference=True, save_as=1, upsampling=upsampling,
                                               save_before_ct=save_before_ct),
                                          dict(crop=SUB, source=1)], SEED)


def shown_alone(upsampling=1):
    """The first frame of the streams above as the only frame of an image, shown."""
    return synth_anim.synth_frames(W, H, [dict(upsampling=upsampling)], SEED)


def noise_still():
    return bench.synth_frame(W, H, SEED, extra=("--noise",))


def noise_with_preview(default_header=False):
    """noise_still() behind a declared 64 x 48 preview: a frame of that size, or with `default_header` a frame of the
    image's size whose all-default frame header takes the image's size."""
    return synth_anim.with_preview(noise_still(), W, H, PREVIEW, default_header)


PREVIEW = (64, 48)
# the first frame of tests/golden/grayscale (a 200 x 200 grey XYB image with an embedded ICC profile) starts here
ICC_HEAD = 245
ICC_SIZE = 200


def icc_image(plan):
    """tests/golden/grayscale's image header and ICC profile, followed by synth_enc frames of `plan` as in
    synth_anim.synth_frames, without durations (the image is not animated)."""
    with open(os.path.join(K.GOLDEN, "grayscale", "input.jxl"), "rb") as f:
        head = f.read()[:ICC_HEAD]
    body = b""
    for i, f in enumerate(plan):
        crop = f.get("crop")
        fw, fh = (crop[2], crop[3]) if crop else (ICC_SIZE, ICC_SIZE)
        body += synth_anim._rewritten_frame(fw, fh, SEED + i, 1.0, animated=False, is_last=i == len(plan) - 1, **f)
    return head + body


ICC_SUB = (40, 30, 100, 80)


STREAMS = {
    "replace_sbct": replace_chain(True),
    "add_onto_sbct": add_onto_slot(True),
    "reference_after_ct": reference_then_crop(),
    "reference_after_ct_up2": reference_then_crop(2),
    "reference_before_ct_up2": reference_then_crop(2, True),
    "preview_small": noise_with_preview(),
    "preview_default_header": noise_with_preview(True),
}
