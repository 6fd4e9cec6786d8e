"""Times jxlb_reconstruct_jpeg on the GPU: end to end over >= 2 s of repeated calls (each returns after a device
synchronise), then one profiled pass that splits device time into the JPEG scan kernels and the HF decode before them,
beside the oracle's single-thread CPU reconstruction of the same input. Needs a CUDA device; prints one JSON line per
input, after the card's name and power limit.

    python tools/jpeg_recon_probe.py [fixture ...]      (default: genshin_ycbcr_420 cafe)
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    return out.strip().splitlines()[0]


def main(names):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_recon_probe needs a CUDA device")
    import jxl_oxide_b200 as J
    import jbr_lib
    jbr_lib.build()  # compiled before anything is timed
    print(json.dumps({"card": card()}), flush=True)
    for name in names:
        data = open(os.path.join(ROOT, "tests", "golden", name, "input.jxl"), "rb").read()
        dec = J.Decoder(0)
        for _ in range(3):
            jpeg = dec.reconstruct_jpeg(data)
        calls, t0 = 0, time.perf_counter()
        while time.perf_counter() - t0 < 2.0:
            dec.reconstruct_jpeg(data)
            calls += 1
        wall_ms = (time.perf_counter() - t0) * 1e3 / calls
        dec.set_profile(1)
        dec.profile_reset()
        dec.reconstruct_jpeg(data)
        per_name = {}
        for n, a, b in dec.timeline():
            if not n.startswith("host:"):
                per_name[n] = per_name.get(n, 0.0) + (b - a)
        dec.set_profile(0)
        jpeg_ms = sum(v for k, v in per_name.items() if k.startswith("jpeg_"))
        hf_ms = sum(v for k, v in per_name.items() if "hf" in k)
        t0 = time.perf_counter()
        ref = jbr_lib.reconstruct_jpeg(data)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        print(json.dumps({
            "input": name, "jpeg_bytes": len(jpeg), "same_as_oracle": jpeg == ref, "calls": calls,
            "gpu_ms_per_call": round(wall_ms, 3), "device_ms_jpeg_kernels": round(jpeg_ms, 3),
            "device_ms_hf_decode": round(hf_ms, 3), "device_ms_by_kernel": {k: round(v, 3) for k, v in sorted(per_name.items())},
            "oracle_single_thread_ms": round(oracle_ms, 1)}), flush=True)


if __name__ == "__main__":
    main(sys.argv[1:] or ["genshin_ycbcr_420", "cafe"])
