"""Times the frame packer (kernels/pack.cu, jxlb_frame_write_ex) on an 8K frame resident in HBM, per layout, sample type
and orientation, and reports the bytes it moves per second against the H100 SXM's 3.35 TB/s HBM3 (data-sheet figure).
Kernel times come from CUDA events around each launch (Decoder.set_profile); the destination is a torch tensor in HBM, so
no host copy is timed. The stream entry point that predates the write specs (jxlb_frame_write_to_device, through
Decoder.frame_to_torch) runs the same kernel and is timed beside it on the same frame.

    python tools/pack_probe.py [--reps 20] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402
import jxl_oxide_b200 as J  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
W, H = 7680, 4320
# colour + alpha + two spot colours + five other extra channels: every selection rule has something to select
EXTRAS = ["alpha:8:0:1", "spot:8:0:1", "spot:8:0:1"] + ["unknown:8:0:1"] * 5
CASES = [("stream", np.uint8), ("stream", np.uint16), ("stream", np.float32), ("stream_no_alpha", np.uint8),
         ("all_channels", np.float32), ("planar", np.float32), ("planar", np.uint8)]


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_ms(dec, name, run, reps):
    for _ in range(3):
        run()
    dec.set_profile(1)
    dec.profile_reset()
    for _ in range(reps):
        run()
    n, ms = dec.profile(name)
    dec.set_profile(0)
    assert n == reps, (name, n)
    return ms / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    data = bench.synth_frame(W, H, 11, extra=tuple(a for e in EXTRAS for a in ("--extra", e)))
    dec = J.Decoder(0)
    dec.decode(data)
    info = dec.frame_info(0)
    spots = 2
    results = []
    for layout, dtype in CASES:
        for orientation in (1, 6):
            spec = J.write_spec(layout, dtype, orientation, True)
            shape, nbytes = dec.frame_write_shape(0, spec)
            nc = shape[0] if layout == "planar" else shape[2]
            tdt = {np.uint8: torch.uint8, np.uint16: torch.uint16, np.float32: torch.float32}[dtype]
            out = torch.empty(shape, dtype=tdt, device="cuda:0")
            ms = kernel_ms(dec, "pack", lambda: dec.frame_write(0, layout, dtype, orientation, out=out), args.reps)
            read_planes = nc + (spots if layout.startswith("stream") else 0)
            moved = W * H * read_planes * 4 + nbytes
            results.append(dict(kernel="pack", entry="frame_write", layout=layout, dtype=np.dtype(dtype).name, orientation=orientation, channels=nc,
                                ms=round(ms, 4), bytes=moved, gb_s=round(moved / ms / 1e6, 1),
                                hbm_share=round(moved / (ms / 1e3) / HBM_BYTES_PER_S, 3)))
            print(json.dumps(results[-1]), flush=True)
    for dtype in (np.uint8, np.uint16):
        for orientation in (1, 6):
            out = dec.frame_to_torch(0, dtype=dtype, orientation=orientation)
            ms = kernel_ms(dec, "pack", lambda: dec.frame_to_torch(0, dtype=dtype, orientation=orientation, out=out), args.reps)
            nc = out.shape[2]
            moved = W * H * (nc + spots) * 4 + out.numel() * out.element_size()
            results.append(dict(kernel="pack", entry="frame_to_torch", layout="stream", dtype=np.dtype(dtype).name,
                                orientation=orientation, channels=nc, ms=round(ms, 4), bytes=moved, gb_s=round(moved / ms / 1e6, 1),
                                hbm_share=round(moved / (ms / 1e3) / HBM_BYTES_PER_S, 3)))
            print(json.dumps(results[-1]), flush=True)
    report = dict(gpu=gpu_name_and_power_limit(), frame=[W, H], channels=info.num_channels, results=results)
    print(json.dumps(dict(gpu=report["gpu"], frame=report["frame"], channels=report["channels"])))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
