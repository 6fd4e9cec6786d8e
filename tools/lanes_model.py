"""SIMT model of the thread-per-stream HF kernel from its host emulation (tests/emu): how full the warps are and how
often the divergent parts of a loop trip run. Usage: python tools/lanes_model.py [file.jxl ...] (default: the 8K
synthetic bench frame and starrail.d1-e6)."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import oracle_lib  # noqa: E402


def model(name, data):
    L = oracle_lib.emu_lib()
    out = (ctypes.c_uint64 * 6)()
    L.jxle_lane_stats(out, 1)
    oracle_lib.OracleImage(data, threads=os.cpu_count() or 1, emu=True).close()
    L.jxle_lane_stats(out, 1)
    streams, symbols, warp_trips, hdr_trips, coef_trips, warps = [int(x) for x in out]
    print(f"{name}: {streams} streams in {warps} warps, {symbols} symbols ({symbols / max(streams, 1):.0f} per stream)")
    print(f"  warp trips {warp_trips} -> {symbols / max(warp_trips, 1):.1f} symbols per trip "
          f"(lane efficiency {symbols / max(warp_trips * 32, 1):.2f}); one-lane-per-warp kernel: {symbols} trips")
    print(f"  trips with a lane on a non-zero count (it may take its next varblock record): {hdr_trips / max(warp_trips, 1):.2f}, "
          f"with a lane on a coefficient: {coef_trips / max(warp_trips, 1):.2f}")


if __name__ == "__main__":
    files = sys.argv[1:]
    if files:
        for f in files:
            model(os.path.basename(f), open(f, "rb").read())
    else:
        model("synth 7680x4320 d1.0 seed 1", bench.synth_frame(7680, 4320, 1))
        model("starrail.d1-e6", open(os.path.join(ROOT, "tests", "golden", "benchmark-data", "starrail.d1-e6.jxl"), "rb").read())
