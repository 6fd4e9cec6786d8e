"""Pipeline experiments (not part of the bench contract): frames/s of the frame pipeline for one workload under a few
settings, and where a frame's wall-clock latency goes (host phases, device waits included).
    python tools/pipe_probe.py synth4k value 32:8 48:10 --phases
"""
import os
import sys
import time

sys.path.insert(0, '.')
import bench  # noqa: E402
import jxl_oxide_b200 as J  # noqa: E402

PHASES = ["lf_global", "alloc", "lf_coeff", "mlf", "hf_metadata", "hf_global", "heavy_wait", "pass_groups", "inverse_transforms",
          "render_vardct", "filters", "filters_colour"]


def main():
    workload, mode = sys.argv[1], sys.argv[2]
    settings = [a for a in sys.argv[3:] if not a.startswith("--")]
    phases = "--phases" in sys.argv
    noaff = "--no-affinity" in sys.argv
    hf = int(os.environ.get("PROBE_HF", "16"))
    nframes = int(os.environ.get("PROBE_FRAMES", "96"))
    _, frames, (w, h) = bench.load_workload(workload, 4)
    for st in settings:
        workers, heavy = (int(x) for x in st.split(":"))
        pipe = J.Pipeline(0, workers=workers, heavy_frames=heavy, hf_streams_per_cta=hf, no_affinity=noaff,
                          batch_streams=int(os.environ.get("PROBE_BATCH", "6")))
        for k, f in enumerate(frames):
            pipe.preload(k, f)

        def run(n):
            sent = got = 0
            while got < n:
                while sent < n and sent - got < 2 * workers + 16:
                    if mode == "value":
                        pipe.submit(slot=sent % len(frames))
                    elif mode == "hostin":    # host bytes in, no output
                        pipe.submit(data=frames[sent % len(frames)])
                    elif mode == "slotout":   # resident input, planar f32 out
                        pipe.submit(slot=sent % len(frames), mode=1)
                    else:
                        pipe.submit(data=frames[sent % len(frames)], mode=1 if mode == "e2e" else 2)
                    sent += 1
                if mode in ("value", "hostin"):
                    pipe.wait()
                else:
                    _, addr, _ = pipe.wait(want_output=True)
                    pipe.release_output(addr)
                got += 1
        run(max(workers, 24))
        decs = [pipe.decoder(i) for i in range(workers)]
        trace = "--trace" in sys.argv
        if phases or trace:
            for d in decs:
                d._L.jxlb_set_profile(d._h, 2 if trace else 3)
                d.profile_reset()
        t = time.perf_counter()
        run(nframes)
        dt = time.perf_counter() - t
        line = "%s %s workers=%d heavy=%d hf=%d: %.1f frames/s, %.0f MP/s, %.2f ms/frame" % (
            workload, mode, workers, heavy, hf, nframes / dt, w * h * nframes / dt / 1e6, dt / nframes * 1e3)
        if phases:
            acc = {}
            for p in PHASES:
                n = sum(d.profile("host:" + p)[0] for d in decs)
                ms = sum(d.profile("host:" + p)[1] for d in decs)
                if n:
                    acc[p] = round(ms / n, 1)
            line += "\n    wall ms per frame by host phase: %s  (sum %.0f)" % (acc, sum(acc.values()))
            # heavy slot: acquire -> grant, grant -> release (ms per frame), and streams taken before begin_heavy_stage()
            slot = {}
            for p in ("slot_wait", "slot_hold"):
                n = sum(d.profile("host:" + p)[0] for d in decs)
                slot[p] = round(sum(d.profile("host:" + p)[1] for d in decs) / n, 1) if n else None
            slot["slot_before_heavy"] = sum(d.profile("host:slot_before_heavy")[0] for d in decs)
            line += "\n    heavy slot: %s" % slot
        if trace:  # per Modular launch: host launch -> device start, device run, device end -> host return
            q, run_ms, wake = [], [], []
            for d in decs:
                tl = d.timeline()
                for k in range(0, len(tl) - 1, 2):
                    (hn, h0, h1), (dn, d0, d1) = tl[k], tl[k + 1]
                    q.append(d0 - h0)
                    run_ms.append(d1 - d0)
                    wake.append(h1 - d1)
            import numpy as np
            if q:
                line += "\n    modular launches %d: launch->start mean %.2f p90 %.2f ms | device run mean %.1f | end->return mean %.2f p90 %.2f ms" % (
                    len(q), np.mean(q), np.percentile(q, 90), np.mean(run_ms), np.mean(wake), np.percentile(wake, 90))
        print(line, flush=True)
        pipe.close()


if __name__ == "__main__":
    main()
