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


def image_header(width, height, animation):
    """synth_enc's image header (sRGB, XYB, 8 bits), with an AnimationHeader (100 ticks/s, no timecodes) if asked."""
    w = BitWriter()
    w.write(16, 0x0AFF)
    w.write(1, 0)  # SizeHeader: not small
    _dim(w, height)
    w.write(3, 0)  # no ratio
    _dim(w, width)
    if not animation:
        w.write(1, 1)  # ImageMetadata all_default
    else:
        w.write(1, 0)  # all_default
        w.write(1, 1)  # extra_fields
        w.write(3, 0)  # orientation 1
        w.write(1, 0)  # have_intrinsic_size
        w.write(1, 0)  # have_preview
        w.write(1, 1)  # have_animation
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


def frame_header(w, crop=None, source=0, duration=1, is_last=False, save_as=0):
    """A regular VarDCT frame header (jxl-frame/src/header.rs:9-134) with default filters, then the TOC's permuted bit.
    `crop` = (x0, y0, width, height) or None for the full canvas; blending is Replace."""
    w.write(1, 0)  # all_default
    w.write(2, 0)  # Regular
    w.write(1, 0)  # VarDCT
    w.write(2, 0)  # flags = 0
    w.write(2, 0)  # upsampling = 1
    w.write(3, 3)  # x_qm_scale
    w.write(3, 2)  # b_qm_scale
    w.write(2, 0)  # num_passes = 1
    w.write(1, 1 if crop else 0)
    if crop:
        x0, y0, cw, ch = crop
        w.u32(CROP, 2 * x0)  # unpack_signed: non-negative offsets are doubled
        w.u32(CROP, 2 * y0)
        w.u32(CROP, cw)
        w.u32(CROP, ch)
    w.write(2, 0)  # blend mode Replace
    if crop:
        w.write(2, source)  # a cropped frame does not reset the canvas: it names its source slot
    w.u32([(0, 0), (1, 0), (0, 8), (0, 32)], duration)
    w.write(1, 1 if is_last else 0)
    resets = crop is None
    if not is_last:
        w.write(2, save_as)
        if resets and (duration == 0 or save_as != 0):
            w.write(1, 0)  # save_before_ct
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


def synth_animation(width, height, frames, mode, seed=1, distance=1.0):
    """Encoded animation: `frames` synth_enc frames of seeds seed, seed + 1, ..."""
    import bench
    plan = frame_plan(mode, frames, width, height)
    head = image_header(width, height, True).bytes()
    body = b""
    for i, (crop, source, duration, save_as) in enumerate(plan):
        fw, fh = (crop[2], crop[3]) if crop else (width, height)
        single = bench.synth_frame(fw, fh, seed + i, distance)
        prefix = image_header(fw, fh, False)
        prefix.pad()
        prefix.write(1, 1)  # the all-default frame header
        prefix.write(1, 0)  # TOC not permuted
        toc_byte = (len(prefix.bits) + 7) // 8
        if prefix.bytes() != single[:toc_byte]:
            raise ValueError("synth_enc no longer writes the layout this tool expects")
        w = BitWriter()
        frame_header(w, crop, source, duration, i == len(plan) - 1, save_as)
        body += w.bytes() + single[toc_byte:]
    return head + body


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
