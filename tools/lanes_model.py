"""SIMT model of the thread-per-stream HF kernel from its host emulation (tests/emu, lanes_k.mk): for each number of streams per
warp (K), how full the warps are and how often the divergent parts of a loop trip run. Usage:
python tools/lanes_model.py [file.jxl ...] (default: the 8K synthetic bench frame and starrail.d1-e6)."""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import oracle_lib  # noqa: E402


KS = (32, 16, 8, 4)
EMU = os.path.join(ROOT, "tests", "emu")


def lanes_k_lib():
    """The HF lanes emulation with the SIMT model of every K (tests/emu/lanes_k.mk)."""
    subprocess.check_call(["make", "-s", "-C", EMU, "-f", "lanes_k.mk"])
    return oracle_lib._load(os.path.join(EMU, "_build", "libjxlemu_lanes_k.so"), None)


def model(name, data):
    L = lanes_k_lib()
    oracle_lib.emu_lib = lambda: L  # OracleImage(..., emu=True) decodes with this build
    out = (ctypes.c_uint64 * 6)()
    for k in KS:
        L.jxle_lane_k_stats(k, out, 1)
    oracle_lib.OracleImage(data, threads=os.cpu_count() or 1, emu=True).close()
    for k in KS:
        L.jxle_lane_k_stats(k, out, 1)
        streams, symbols, warp_trips, hdr_trips, coef_trips, warps = [int(x) for x in out]
        if k == KS[0]:
            print(f"{name}: {streams} streams, {symbols} symbols ({symbols / max(streams, 1):.0f} per stream); "
                  f"one-lane-per-warp kernel: {symbols} trips")
        print(f"  K={k:2d}: {warps} warps, {warp_trips} warp trips -> {symbols / max(warp_trips, 1):.1f} symbols per trip "
              f"(lane efficiency {symbols / max(warp_trips * k, 1):.2f}), {warp_trips / max(warps, 1):.0f} trips per warp; "
              f"trips with a lane on a non-zero count {hdr_trips / max(warp_trips, 1):.2f}, "
              f"on a coefficient {coef_trips / max(warp_trips, 1):.2f}")


if __name__ == "__main__":
    files = sys.argv[1:]
    if files:
        for f in files:
            model(os.path.basename(f), open(f, "rb").read())
    else:
        model("synth 7680x4320 d1.0 seed 1", bench.synth_frame(7680, 4320, 1))
        model("starrail.d1-e6", open(os.path.join(ROOT, "tests", "golden", "benchmark-data", "starrail.d1-e6.jxl"), "rb").read())
