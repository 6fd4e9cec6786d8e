"""Streams per warp of the thread-per-stream HF kernel without a GPU: the setter's argument checks, and the host
emulation's SIMT model (tests/emu/lanes_k_emu.cc), which groups K consecutive streams of the launch order into a warp as
the device does. The device launch itself is covered by tests/test_zz_gpu_hf_packing.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import bench
import jxl_oxide_b200
import oracle_lib


def test_set_hf_streams_per_warp_rejects_bad_arguments():
    L = ctypes.CDLL(jxl_oxide_b200.LIB_PATH)
    L.jxlb_set_hf_streams_per_warp.argtypes = [ctypes.c_void_p, ctypes.c_int32]
    L.jxlb_set_hf_streams_per_warp.restype = ctypes.c_int32
    for k in (0, 4, 8, 16, 32, -1, 1, 2, 12, 64, 128):
        assert L.jxlb_set_hf_streams_per_warp(None, k) == jxl_oxide_b200.ERR_INVALID_ARG
    assert "jxlb_set_hf_streams_per_warp" in jxl_oxide_b200.EXPORTED_SYMBOLS


EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
KS = (32, 16, 8, 4)


@pytest.fixture
def lanes_k(monkeypatch):
    """OracleImage(..., emu=True) decodes with the build of the emulation that models every K (tests/emu/lanes_k.mk)."""
    subprocess.check_call(["make", "-s", "-C", EMU, "-f", "lanes_k.mk"])
    L = oracle_lib._load(os.path.join(EMU, "_build", "libjxlemu_lanes_k.so"), None)
    monkeypatch.setattr(oracle_lib, "emu_lib", lambda: L)
    return L


def test_lane_model_follows_streams_per_warp(lanes_k):
    L = lanes_k
    out = (ctypes.c_uint64 * 6)()
    for k in KS:
        L.jxle_lane_k_stats(k, out, 1)
    data = bench.synth_frame(2000, 1500, 3)  # 48 streams, one decode_hf launch
    img = oracle_lib.OracleImage(data, threads=4, capture=True, emu=True)
    want = oracle_lib.OracleImage(data, threads=4, capture=True)
    assert np.array_equal(img.frame(0)[0].view(np.uint32), want.frame(0)[0].view(np.uint32))
    img.close()
    want.close()
    stats = {}
    for k in KS:
        L.jxle_lane_k_stats(k, out, 1)
        stats[k] = [int(x) for x in out]  # streams, symbols, warp trips, trips on a count, trips on a coefficient, warps
    streams, symbols = stats[32][0], stats[32][1]
    assert streams == 48 and symbols > 0
    for k, (n, sym, trips, hdr, coef, warps) in stats.items():
        assert (n, sym) == (streams, symbols)  # the same streams decode the same symbols whatever the packing
        assert warps == -(-streams // k)
        assert symbols / k <= trips <= symbols  # a warp trip carries between one and K symbols
        assert max(hdr, coef) <= trips <= hdr + coef
    # fewer streams per warp: more warps, so more warp trips in all
    assert stats[4][2] >= stats[8][2] >= stats[16][2] >= stats[32][2]
