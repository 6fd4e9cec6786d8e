"""Host emulation of the Modular stream kernel (kernels/modular_lanes.cuh).

tests/emu/modular_emu.cc compiles the per-stream code of modular_stream_kernel for the host -- the channel dispatch,
the general loop, the single-leaf loop and the weighted predictor's fast loop with its row prologue -- and plugs it
into the oracle's planner in place of the oracle's own Modular decoder. It decodes launches built by the CUDA backend's
own table code (launch_tables.cc): compacted and shared channel subtrees by default, the whole-tree plans when the node
limit is lowered to 0. Decoded samples reach every pixel, and a wrong end position breaks the parse of what follows the
stream, so equal frames pin both. The LF shapes include channels 1, 2 and 129 samples wide (a last prologue chunk of
one column) and rows of 1 and 2 samples, and a forced range trip runs the fast loop's fallback. The device launch
itself is covered by the GPU parity tests.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import bench
import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
GOLDEN = os.path.join(ROOT, "tests", "golden")
SRCS = ["modular_emu.cc", "launch_tables_host.cc"] + [os.path.join("..", "..", "oracle", f) for f in
                             ("oracle_capi.cc", "oracle_modular.cc", "oracle_vardct.cc", "oracle_render.cc")] + \
       [os.path.join("..", "..", "jxl_oxide_b200", "csrc", "host", f) for f in
        ("entropy.cc", "headers.cc", "modular_syntax.cc", "frame_syntax.cc", "planner.cc", "icc.cc")]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("modular_emu") / "libjxlmodemu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                           "-I/usr/local/cuda/include", "-DJXLO_BACKEND_FACTORY=make_modular_emu_backend", "-shared",
                           "-Wl,-Bsymbolic", "-o", out] + SRCS, cwd=EMU)
    L = oracle_lib._load(out, None)
    L.jxlme_stats.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]
    L.jxlme_force_trip.argtypes = [ctypes.c_uint64]
    L.jxlme_max_channel_tree_nodes.argtypes = [ctypes.c_uint64]
    L.jxlme_max_channel_tree_nodes.restype = ctypes.c_uint64
    return L


# [0] streams, [1] fast-loop channels, [2] of those decoded again after a range trip, [3] single-leaf channels,
# [4] jobs built compact, [5] jobs built with the whole-tree plans, [6] channels sharing an earlier channel's subtree,
# [7] jobs of launches without the fast loop (a table not staged)
def _stats(L):
    v = (ctypes.c_uint64 * 8)()
    L.jxlme_stats(v, 1)
    return list(v)


def _decode(L, data):
    saved = oracle_lib._EMU_LIB
    oracle_lib._EMU_LIB = L
    try:
        return oracle_lib.OracleImage(data, threads=4, emu=True)
    finally:
        oracle_lib._EMU_LIB = saved


def _same(L, data, whole_tree=False):
    _stats(L)
    want = oracle_lib.OracleImage(data, threads=4)
    if whole_tree:
        limit = L.jxlme_max_channel_tree_nodes(0)
        try:
            got = _decode(L, data)
        finally:
            L.jxlme_max_channel_tree_nodes(limit)
    else:
        got = _decode(L, data)
    stats = _stats(L)
    assert stats[0] > 0, "the emulated Modular path did not run"
    assert stats[4] + stats[5] == stats[0]
    if whole_tree:
        assert stats[5] > 0, "no job was built with the whole-tree plans"
    else:
        assert stats[4] == stats[0], "a job was not built with compacted channel subtrees"
    assert got.num_frames == want.num_frames
    for i in range(want.num_frames):
        a, b = want.frame(i)[0], got.frame(i)[0]
        assert a.shape == b.shape
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"frame {i} differs"
    return stats


# LF channels (1/8 of the frame per axis, 256 x 256 per LF group): 3080 x 2064 -> widths 256 and 129, heights 256 and 2;
# 2056 x 600 -> widths 256 and 1; 3840 x 2160 is the 4K bench frame
@pytest.mark.parametrize("w,h", [(3080, 2064), (2056, 600), (3840, 2160)])
def test_emulated_modular_streams_match_oracle_on_synthetic_frames(emu, w, h):
    stats = _same(emu, bench.synth_frame(w, h, 3))
    assert stats[1] > 0, "no channel took the weighted-predictor fast loop"
    assert stats[3] > 0, "no channel took the single-leaf loop"
    assert stats[2] == 0


@pytest.mark.parametrize("trip_at", [1, 300, 5000])
def test_emulated_fast_loop_fallback_after_range_trip(emu, trip_at):
    # the fast loop reports a range trip once a channel has this many samples; the channel is decoded again by the
    # general loop from the stream state at its start
    emu.jxlme_force_trip(trip_at)
    try:
        stats = _same(emu, bench.synth_frame(3080, 2064, 5))
    finally:
        emu.jxlme_force_trip(0)
    assert stats[2] > 0
    if trip_at == 1:  # every channel reaches one sample
        assert stats[2] == stats[1]


def test_emulated_modular_streams_match_oracle_on_synthetic_modular_frame(emu):
    stats = _same(emu, bench.synth_frame(1000, 600, 7, extra=("--modular",)))
    assert stats[6] > 0, "no channels shared a subtree copy"


FIXTURES = ["grayalpha", "squeeze_edge", "issue_311", "patches_lossless", "lossless_pfm", "lz77_flower", "delta_palette"]


def _fixture(name):
    d = os.path.join(GOLDEN, name)
    return open(os.path.join(d, sorted(f for f in os.listdir(d) if f.endswith(".jxl"))[0]), "rb").read()


@pytest.mark.parametrize("name", FIXTURES)
def test_emulated_modular_streams_match_oracle_on_fixture(emu, name):
    stats = _same(emu, _fixture(name))
    if name == "squeeze_edge":  # a Squeeze image's channels under one tree that never tests the channel index
        assert stats[6] > 0, "no channels shared a subtree copy"
    if name == "lz77_flower":  # the LZ77 window lives in global memory: the launch is not all staged
        assert stats[7] == stats[0] and stats[1] == 0, "the fast loop was not disabled"


# Node limit 0: every job with a channel subtree of more than one node walks the frame's whole tree (single-leaf channels
# still compact, so squeeze_edge keeps every job compact).
@pytest.mark.parametrize("name", [n for n in FIXTURES if n != "squeeze_edge"] + ["synthetic"])
def test_emulated_modular_streams_match_oracle_with_whole_tree_plans(emu, name):
    _same(emu, bench.synth_frame(2056, 600, 3) if name == "synthetic" else _fixture(name), whole_tree=True)
