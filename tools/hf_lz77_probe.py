"""What LZ77 in the HF coefficient streams costs on the device (not part of the bench contract).

One 7680x4320 synthetic frame (tools/synth_enc.cc, seed 1) in three codings of the same coefficients: plain, --hf-lz77
rle and --hf-lz77 match. Times decode_hf (CUDA events, jxlb_profile_get) and the whole decode (host clock around
decode + sync), the codings alternated rep by rep. A plain frame runs the default schedule (one warp per stream, 16 per
CTA); it is also timed at 128 streams per CTA, the thread-per-stream schedule every LZ77 frame runs. With --ycbcr MODE
the frame is a chroma-subsampled one laid out like a JPEG transcode (synth_enc --ycbcr: Cb, Y, Cr, DCT8 everywhere).
With --file PATH the frames are that file and its HF passes restreamed with rle and match codes (tools/hf_restream.cc).

    python tools/hf_lz77_probe.py [--reps 10] [--seed 1] [--ycbcr 444|420|422|440 | --file PATH]
"""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import jxl_oxide_b200 as J  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--ycbcr", choices=["444", "420", "422", "440"])
    ap.add_argument("--file")
    a = ap.parse_args()
    w, h = 7680, 4320
    extra = ["--ycbcr", a.ycbcr] if a.ycbcr else []
    if a.file:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import hf_restream
        with open(a.file, "rb") as f:
            frames = {"plain": f.read()}
        for mode in ("rle", "match"):
            frames[mode], copied = hf_restream.restream(frames["plain"], mode)
            print(f"{mode}: {copied} values copied")
    else:
        frames = {"plain": bench.synth_frame(w, h, a.seed, extra=tuple(extra))}
    with tempfile.TemporaryDirectory() as tmp:
        for mode in () if a.file else ("rle", "match"):
            out = os.path.join(tmp, f"{mode}.jxl")
            r = subprocess.run([bench.synth_tool(), "--width", str(w), "--height", str(h), "--seed", str(a.seed), "-o", out,
                                "--hf-lz77", mode] + extra, capture_output=True, text=True, check=True)
            print(r.stderr.strip().splitlines()[-1])
            frames[mode] = open(out, "rb").read()
    runs = [("plain", 0), ("plain", 128), ("rle", 0), ("match", 0)]
    d = J.Decoder(0)
    for name, spc in runs:  # warm-up: module loads, pool growth
        d.set_hf_streams_per_cta(spc)
        for _ in range(2):
            d.decode(frames[name])
            d.sync()
            d.release_frames()
    d.set_profile(True)
    hf = {r: [] for r in runs}
    total = {r: [] for r in runs}
    for _ in range(a.reps):
        for r in runs:
            name, spc = r
            d.set_hf_streams_per_cta(spc)
            d.profile_reset()
            t = time.perf_counter()
            d.decode(frames[name])
            d.sync()
            total[r].append((time.perf_counter() - t) * 1e3)
            hf[r].append(d.profile("decode_hf")[1])
            d.release_frames()
    d.close()
    what = a.file or f"{w}x{h}{' YCbCr ' + a.ycbcr if a.ycbcr else ''}, seed {a.seed}"
    print(f"card: {card()}; {what}, {a.reps} reps each, alternated; median [min .. max] ms")
    for r in runs:
        name, spc = r
        print(f"  {name:5s} streams/CTA {spc or 'default':>7}: {len(frames[name]) / 1e6:6.2f} MB  decode_hf "
              f"{statistics.median(hf[r]):6.2f} [{min(hf[r]):.2f} .. {max(hf[r]):.2f}]  whole decode "
              f"{statistics.median(total[r]):6.2f} [{min(total[r]):.2f} .. {max(total[r]):.2f}]")


if __name__ == "__main__":
    main()
