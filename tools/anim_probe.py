"""Keyframes per second and HBM high-water of animations through the frame pipeline (jxlb_pipeline_submit_keyframes),
against the same frames submitted as separate single-frame images (jxlb_pipeline_submit).

Animations are synthetic (tools/synth_anim.py) at 3840x2160: `independent` (one segment per keyframe, spread over the
workers) and `chain` (one segment: one worker renders every keyframe in order). Outputs are decoded in HBM and released
(out mode 0), so the numbers are decode rates. HBM high-water is the device's used memory (cudaMemGetInfo, sampled
every 2 ms) above what it was before the pipeline was created. Prints one JSON line per case; needs a GPU.

    python tools/anim_probe.py --frames 32 64 --workers 16 --heavy 8
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import synth_anim  # noqa: E402


class HbmSampler:
    def __init__(self, torch):
        self.torch = torch
        self.base = self._used()
        self.peak = self.base
        self._stop = False
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def _used(self):
        free, total = self.torch.cuda.mem_get_info(0)
        return total - free

    def _run(self):
        while not self._stop:
            self.peak = max(self.peak, self._used())
            time.sleep(0.002)

    def stop(self):
        self._stop = True
        self._t.join()
        return (self.peak - self.base) / 2**20


def run(J, torch, submit, count, workers, heavy, reps):
    """Best keyframes/s over `reps` timed passes after one warm-up pass, and the HBM high-water in MiB."""
    hbm = HbmSampler(torch)
    pipe = J.Pipeline(0, workers=workers, heavy_frames=heavy)
    best = 0.0
    for rep in range(reps + 1):
        t0 = time.perf_counter()
        submit(pipe)
        while pipe.in_flight:
            pipe.wait_keyframe()
        dt = time.perf_counter() - t0
        if rep:
            best = max(best, count / dt)
    pipe.close()
    return best, hbm.stop()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--modes", nargs="+", default=["independent", "chain"])
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--workers", type=int, default=16)
    ap.add_argument("--heavy", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    import jxl_oxide_b200 as J
    if not torch.cuda.is_available():
        sys.exit("anim_probe needs a GPU")
    props = torch.cuda.get_device_properties(0)
    gpu = {"name": props.name}
    try:
        import subprocess
        gpu["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers still stand, without the card's limits
        gpu["power_limit"] = f"unavailable: {e}"
    print(json.dumps({"gpu": gpu}), flush=True)
    for mode in a.modes:
        for n in a.frames:
            data = synth_anim.synth_animation(a.width, a.height, n, mode)
            plan = synth_anim.frame_plan(mode, n, a.width, a.height)
            singles = [bench.synth_frame(c[2] if c else a.width, c[3] if c else a.height, 1 + i) for i, (c, *_rest) in enumerate(plan)]
            kps, hbm = run(J, torch, lambda p: p.submit_keyframes(data), n, a.workers, a.heavy, a.reps)
            fps, hbm1 = run(J, torch, lambda p: [p.submit(s) for s in singles], n, a.workers, a.heavy, a.reps)
            nk, ns, _ = J.image_keyframes(data)
            print(json.dumps({"mode": mode, "keyframes": nk, "segments": ns, "size": [a.width, a.height],
                              "workers": a.workers, "heavy_frames": a.heavy,
                              "animation_keyframes_per_s": round(kps, 2), "animation_hbm_high_water_mib": round(hbm, 1),
                              "separate_images_per_s": round(fps, 2), "separate_hbm_high_water_mib": round(hbm1, 1)}), flush=True)


if __name__ == "__main__":
    main()
