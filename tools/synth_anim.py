"""Synthetic animations: frames of tools/synth_enc.cc (VarDCT, one seed per frame) put behind an animated image header
and frame headers that set the duration, crop, blending source and reference slot of each frame.

A synth_enc stream with default options is the image header, padding, a one-bit all-default frame header, the TOC's
`permuted` bit, padding, and then the byte-aligned TOC and sections. The frame header is rewritten here; the TOC and the
sections are taken over byte for byte.

Frame modes:
- independent: full-canvas Replace frames, duration 1: one segment per keyframe.
- chain: a full-canvas first frame, then frames that replace a sub-rectangle of the canvas kept in slot 1 and save the
  result to slot 1, GIF style: one segment.
- mixed: a full-canvas frame every 3 frames that starts a new chain; frame 1 has duration 0 (composed into the next
  keyframe), and the last frame of each chain saves to slot 2, which no frame reads.

Frame kinds (synth_frames): each frame of a plan may also be saved before the colour transform, be a reference-only
frame (optionally upsampled: its synth_enc frame is coded at the reduced size), or blend with Add onto its source slot.
`with_preview` puts a preview frame in front of a still synth_enc stream.

    python tools/synth_anim.py --width 3840 --height 2160 --frames 32 --mode independent -o anim.jxl
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class BitWriter:
    def __init__(self):
        self.bits = []

    def write(self, n, v):
        for i in range(n):
            self.bits.append((v >> i) & 1)

    def u32(self, dists, v):
        """U32 with distributions [(offset, bits)] x 4: the first one that can hold v."""
        for sel, (off, nb) in enumerate(dists):
            if v >= off and v - off < (1 << nb) if nb else v == off:
                self.write(2, sel)
                self.write(nb, v - off)
                return
        raise ValueError(f"{v} does not fit {dists}")

    def pad(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def bytes(self):
        self.pad()
        return bytes(sum(b << i for i, b in enumerate(self.bits[k:k + 8])) for k in range(0, len(self.bits), 8))


def _dim(w, v):  # synth_enc's SizeHeader dimension
    if v <= 512:
        w.write(2, 0), w.write(9, v - 1)
    elif v <= 8192:
        w.write(2, 1), w.write(13, v - 1)
    else:
        w.write(2, 2), w.write(18, v - 1)


def _preview_dim(w, v):  # PreviewHeader dimension without div8 (jxl-image/src/lib.rs:172-187)
    for sel, (off, nb) in enumerate([(1, 6), (65, 8), (321, 10), (1345, 12)]):
        if off <= v < off + (1 << nb):
            w.write(2, sel), w.write(nb, v - off)
            return
    raise ValueError(v)


def image_header(width, height, animation, preview=None):
    """synth_enc's image header (sRGB, XYB, 8 bits), with an AnimationHeader (100 ticks/s, no timecodes) if asked and a
    preview of `preview` = (width, height) if given."""
    w = BitWriter()
    w.write(16, 0x0AFF)
    w.write(1, 0)  # SizeHeader: not small
    _dim(w, height)
    w.write(3, 0)  # no ratio
    _dim(w, width)
    if not animation and not preview:
        w.write(1, 1)  # ImageMetadata all_default
    else:
        w.write(1, 0)  # all_default
        w.write(1, 1)  # extra_fields
        w.write(3, 0)  # orientation 1
        w.write(1, 0)  # have_intrinsic_size
        w.write(1, 1 if preview else 0)  # have_preview
        if preview:
            w.write(1, 0)  # div8
            _preview_dim(w, preview[1])
            w.write(3, 0)  # no ratio
            _preview_dim(w, preview[0])
        w.write(1, 1 if animation else 0)  # have_animation
        if animation:
            w.write(2, 0)  # tps_numerator = 100
            w.write(2, 0)  # tps_denominator = 1
            w.write(2, 0)  # num_loops = 0
            w.write(1, 0)  # have_timecodes
        w.write(1, 0)  # integer samples
        w.write(2, 0)  # 8 bits
        w.write(1, 1)  # modular_16bit_buffers
        w.write(2, 0)  # no extra channels
        w.write(1, 1)  # xyb_encoded
        w.write(1, 1)  # ColourEncoding all_default
        w.write(1, 1)  # ToneMapping all_default
        w.write(2, 0)  # extensions
    w.write(1, 1)  # default_m
    return w


CROP = [(0, 8), (256, 11), (2304, 14), (18688, 30)]


def frame_header(w, crop=None, source=0, duration=1, is_last=False, save_as=0, add=False, save_before_ct=False,
                 reference=False, upsampling=1, animated=True):
    """A regular VarDCT frame header (jxl-frame/src/header.rs:9-134) with default filters, then the TOC's permuted bit.
    `crop` = (x0, y0, width, height) or None for the full canvas; blending is Replace, or Add with `add`. A `reference`
    frame is reference-only: it has no offset, blending, duration or is_last, and always signals save_before_ct."""
    w.write(1, 0)  # all_default
    w.write(2, 2 if reference else 0)  # ReferenceOnly / Regular
    w.write(1, 0)  # VarDCT
    w.write(2, 0)  # flags = 0
    w.write(2, {1: 0, 2: 1, 4: 2, 8: 3}[upsampling])
    w.write(3, 3)  # x_qm_scale
    w.write(3, 2)  # b_qm_scale
    if not reference:
        w.write(2, 0)  # num_passes = 1
    w.write(1, 1 if crop else 0)
    if crop:
        x0, y0, cw, ch = crop
        if not reference:
            w.u32(CROP, 2 * x0)  # unpack_signed: non-negative offsets are doubled
            w.u32(CROP, 2 * y0)
        w.u32(CROP, cw)
        w.u32(CROP, ch)
    resets = crop is None and not add
    if not reference:
        w.write(2, 1 if add else 0)  # blend mode Add / Replace
        if not resets:
            w.write(2, source)  # a frame that does not reset the canvas names its source slot
        if animated:
            w.u32([(0, 0), (1, 0), (0, 8), (0, 32)], duration)
        w.write(1, 1 if is_last else 0)
    if reference or not is_last:
        w.write(2, save_as)
        if reference or (resets and (duration == 0 or save_as != 0)):
            w.write(1, 1 if save_before_ct else 0)
        elif save_before_ct:
            raise ValueError("save_before_ct is signalled only by frames that reset the canvas and are saved")
    w.write(2, 0)  # name: empty
    w.write(1, 1)  # restoration filter all_default
    w.write(2, 0)  # extensions
    w.write(1, 0)  # TOC not permuted
    w.pad()


def frame_plan(mode, n, width, height):
    """[(crop or None, source, duration, save_as)] per frame."""
    sub = (width // 4, height // 4, max(width // 2, 8), max(height // 2, 8))
    plan = []
    for i in range(n):
        if mode == "independent":
            plan.append((None, 0, 1, 0))
        elif mode == "chain":
            plan.append((None, 0, 1, 1) if i == 0 else (sub, 1, 1, 1))
        elif mode == "mixed":
            starts = i % 3 == 0
            ends = i % 3 == 2 or i == n - 1
            duration = 0 if i == 1 else 1
            save = 2 if ends else 1
            plan.append((None, 0, duration, save) if starts else (sub, 1, duration, save))
        else:
            raise ValueError(mode)
    return plan


def _rewritten_frame(fw, fh, seed, distance, animated=True, **header):
    """synth_enc's frame of seed `seed` at fw x fh behind a rewritten frame header."""
    import bench
    single = bench.synth_frame(fw, fh, seed, distance)
    prefix = image_header(fw, fh, False)
    prefix.pad()
    prefix.write(1, 1)  # the all-default frame header
    prefix.write(1, 0)  # TOC not permuted
    toc_byte = (len(prefix.bits) + 7) // 8
    if prefix.bytes() != single[:toc_byte]:
        raise ValueError("synth_enc no longer writes the layout this tool expects")
    w = BitWriter()
    frame_header(w, animated=animated, **header)
    return w.bytes() + single[toc_byte:]


def synth_frames(width, height, plan, seed=1, distance=1.0):
    """Encoded animation of one synth_enc frame per plan entry (seeds seed, seed + 1, ...). An entry holds frame_header's
    keyword arguments; is_last is set on the last entry. A frame is coded at its crop's size, divided by its upsampling."""
    head = image_header(width, height, True).bytes()
    body = b""
    for i, f in enumerate(plan):
        crop, up = f.get("crop"), f.get("upsampling", 1)
        fw, fh = (crop[2], crop[3]) if crop else (width, height)
        body += _rewritten_frame(-(-fw // up), -(-fh // up), seed + i, distance, is_last=i == len(plan) - 1, **f)
    return head + body


def synth_animation(width, height, frames, mode, seed=1, distance=1.0):
    """Encoded animation: `frames` synth_enc frames of seeds seed, seed + 1, ..."""
    plan = frame_plan(mode, frames, width, height)
    return synth_frames(width, height, [dict(crop=crop, source=source, duration=duration, save_as=save_as)
                                        for crop, source, duration, save_as in plan], seed, distance)


def with_preview(still, width, height, preview, default_header=False, preview_seed=99):
    """`still` (a synth_enc stream of width x height whose metadata is all-default) with a preview of `preview` =
    (width, height) declared in the image header and a preview frame in front: a synth_enc frame of that size behind a
    cropped frame header, or with `default_header` a frame of the image's size behind an all-default frame header,
    whose size defaults to the image's and not to the declared preview size (jxl-frame/src/header.rs:51-58)."""
    import bench
    head = image_header(width, height, False).bytes()
    if still[:len(head)] != head:
        raise ValueError("synth_enc no longer writes the layout this tool expects")
    if default_header:
        pframe = bench.synth_frame(width, height, preview_seed)[len(head):]
    else:
        pframe = _rewritten_frame(preview[0], preview[1], preview_seed, 1.0, animated=False, crop=(0, 0) + tuple(preview),
                                  is_last=True)
    return image_header(width, height, False, preview=preview).bytes() + pframe + still[len(head):]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--mode", default="independent", choices=["independent", "chain", "mixed"])
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--distance", type=float, default=1.0)
    ap.add_argument("-o", "--out", required=True)
    a = ap.parse_args()
    with open(a.out, "wb") as f:
        f.write(synth_animation(a.width, a.height, a.frames, a.mode, a.seed, a.distance))


if __name__ == "__main__":
    main()
