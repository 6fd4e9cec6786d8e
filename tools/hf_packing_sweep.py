"""Streams per warp of the pipeline's thread-per-stream HF decoder (jxlb_set_hf_streams_per_warp), measured on one GPU.

For each K: pipeline frames/s with the bench's defaults (64 workers, 16 heavy slots, 128 HF streams per CTA, inputs
resident), `decode_hf` per frame under that load and alone on the GPU (CUDA events, as bench.py takes them), and the heavy
slot's hold and wait per frame (host clock, as tools/pipe_probe.py --phases). The K values are taken in turn, `--rounds`
times over, on one pipeline. With `--parent DIR --bench-runs N`, bench.py's `value` of DIR's build and of this tree,
alternated N times. Prints the card's name, power limit and max SM clock first, and everything as JSON at the end.
    python tools/hf_packing_sweep.py --ks 32,16,8,4 --rounds 2 --parent ab_old --bench-runs 4 [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")  # as bench.py
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "nvidia-smi: n/a"


def sweep(args):
    import bench
    import jxl_oxide_b200 as J
    _, frames, _ = bench.load_workload(args.workload, 4)
    pipe = J.Pipeline(0, workers=64, heavy_frames=16, hf_streams_per_cta=128)
    for k, f in enumerate(frames):
        pipe.preload(k, f)
    decs = [pipe.decoder(i) for i in range(pipe.workers())]

    def run(n):
        sent = got = 0
        while got < n:
            while sent < n and sent - got < 2 * len(decs):
                pipe.submit(slot=sent % len(frames))
                sent += 1
            pipe.wait()
            got += 1

    def counters(level, n):
        for d in decs:
            d._L.jxlb_set_profile(d._h, level)
            d.profile_reset()
        run(n)
        acc = {}
        for name in ("decode_hf", "host:slot_hold", "host:slot_wait"):
            acc[name] = (sum(d.profile(name)[0] for d in decs), sum(d.profile(name)[1] for d in decs))
        for d in decs:
            d._L.jxlb_set_profile(d._h, 0)
        return acc

    ks = [int(k) for k in args.ks.split(",")]
    res = {k: {"frames_per_s": [], "decode_hf_ms_load": [], "decode_hf_ms_solo": [], "slot_hold_ms": [], "slot_wait_ms": []}
           for k in ks}
    for r in range(args.rounds):
        for k in (ks if r % 2 == 0 else ks[::-1]):
            for d in decs:
                d.set_hf_streams_per_warp(k)
            run(args.frames // 2)  # warm-up at this K
            t = time.perf_counter()
            run(args.frames)
            res[k]["frames_per_s"].append(args.frames / (time.perf_counter() - t))
            acc = counters(3, args.frames)
            res[k]["slot_hold_ms"].append(acc["host:slot_hold"][1] / max(acc["host:slot_hold"][0], 1))
            res[k]["slot_wait_ms"].append(acc["host:slot_wait"][1] / max(acc["host:slot_wait"][0], 1))
            acc = counters(1, args.frames)
            res[k]["decode_hf_ms_load"].append(acc["decode_hf"][1] / max(acc["decode_hf"][0], 1))
            for d in decs:
                d._L.jxlb_set_profile(d._h, 1)
                d.profile_reset()
            for _ in range(3):  # one frame at a time: alone on the GPU
                pipe.submit(slot=0)
                pipe.wait()
            n = sum(d.profile("decode_hf")[0] for d in decs)
            res[k]["decode_hf_ms_solo"].append(sum(d.profile("decode_hf")[1] for d in decs) / max(n, 1))
            for d in decs:
                d._L.jxlb_set_profile(d._h, 0)
            print("K=%2d round %d: %.1f frames/s, decode_hf %.2f ms/frame under load, %.2f alone, slot hold %.1f ms, wait %.1f ms" % (
                k, r, res[k]["frames_per_s"][-1], res[k]["decode_hf_ms_load"][-1], res[k]["decode_hf_ms_solo"][-1],
                res[k]["slot_hold_ms"][-1], res[k]["slot_wait_ms"][-1]), flush=True)
    pipe.close()
    return res


def bench_value(tree, workload):
    out = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3",
                          "--no-cpu-baseline", "--workload", workload], capture_output=True, text=True, cwd=tree)
    for line in reversed(out.stdout.splitlines()):
        if line.startswith("{"):
            return json.loads(line)
    raise RuntimeError("bench.py in %s printed no result: %s" % (tree, out.stderr[-2000:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="32,16,8,4")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--frames", type=int, default=192)
    ap.add_argument("--workload", default="synth8k")
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--parent", default=None, help="tree of the build to compare bench.py against")
    ap.add_argument("--bench-runs", type=int, default=0)
    ap.add_argument("--bench-workloads", default="synth8k")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = gpu_info()
    print("GPU (name, power limit, max SM clock):", info, flush=True)
    result = {"gpu": info}
    if not args.no_sweep:
        res = sweep(args)
        result["sweep"] = {str(k): v for k, v in res.items()}
        for k, v in res.items():
            print("K=%2d median: %.1f frames/s, decode_hf %.2f ms under load, %.2f alone, slot hold %.1f ms" % (
                k, statistics.median(v["frames_per_s"]), statistics.median(v["decode_hf_ms_load"]),
                statistics.median(v["decode_hf_ms_solo"]), statistics.median(v["slot_hold_ms"])), flush=True)
    if args.parent and args.bench_runs:
        result["bench"] = {}
        for wl in args.bench_workloads.split(","):
            vals = {"parent": [], "this": []}
            for i in range(args.bench_runs):
                for name, tree in (("parent", os.path.abspath(args.parent)), ("this", ROOT)):
                    t = time.perf_counter()
                    r = bench_value(tree, wl)
                    vals[name].append(r["value"])
                    print("%s %s run %d: value %.1f (%.0f s)" % (wl, name, i, r["value"], time.perf_counter() - t), flush=True)
            result["bench"][wl] = vals
            mp, mt = statistics.median(vals["parent"]), statistics.median(vals["this"])
            spread = {n: (max(v) - min(v)) / statistics.median(v) for n, v in vals.items()}
            print("%s value median: this %.1f (%.1f-%.1f), parent %.1f (%.1f-%.1f): %+.1f %%; spread this %.1f %%, parent %.1f %%" % (
                wl, mt, min(vals["this"]), max(vals["this"]), mp, min(vals["parent"]), max(vals["parent"]),
                100 * (mt / mp - 1), 100 * spread["this"], 100 * spread["parent"]), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
