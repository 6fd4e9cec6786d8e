"""Host emulation of the thread-per-stream HF coefficient kernel (kernels/hf_lanes.cuh).

The per-stream function every device thread runs is plain integer C++ without cross-lane traffic, so
tests/emu/ compiles it for the host and plugs it into the oracle's planner in place of the oracle's own
HF decoder. These tests pin its LOGIC (state machine, contexts, stores, end positions) against the oracle on
every VarDCT shape the fixtures hold; the device launch itself (shared-memory staging, lane interleave) is
covered by tests/test_zz_gpu_schedules.py::test_hf_lanes_* on a GPU.
"""
import ctypes
import os

import numpy as np
import pytest

import bench
import oracle_lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

VARDCT_FIXTURES = [
    "opsin_inverse",        # plain XYB VarDCT, ANS
    "bike",                 # patches + reference frames
    "noise",
    "upsampling",
    "cafe",                 # JPEG transcode 4:2:0: shifted channel grids (SUB path)
    "issue_425",            # 4:2:0 with an odd block count
    "genshin_ycbcr_420",    # 4:2:0 at 2560 x 1440: 60 groups, two warps of streams
    "bench_oriented_brg",   # JPEG transcode 4:4:4
    "grayscale_jpeg",
    "minecraft_vardct_e7",
    "progressive",          # several passes: first pass stores, later passes accumulate
]


def _input(name):
    d = os.path.join(GOLDEN, name)
    for f in sorted(os.listdir(d)):
        if f.endswith(".jxl"):
            return open(os.path.join(d, f), "rb").read()
    raise FileNotFoundError(name)


def _streams():
    L = oracle_lib.emu_lib()
    L.jxle_hf_streams.restype = ctypes.c_uint64
    return L.jxle_hf_streams()


def _same(data, **kw):
    before = _streams()
    want = oracle_lib.OracleImage(data, threads=4, capture=True, **kw)
    got = oracle_lib.OracleImage(data, threads=4, capture=True, emu=True, **kw)
    assert _streams() > before, "the emulated HF path did not run"
    assert got.num_frames == want.num_frames
    for i in range(want.num_frames):
        a, b = want.frame(i)[0], got.frame(i)[0]
        assert a.shape == b.shape
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"frame {i} differs"
    ca, cb = want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32)
    assert len(ca) == len(cb)
    for x, y in zip(ca, cb):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("name", VARDCT_FIXTURES)
def test_emulated_lanes_match_oracle_on_fixture(name):
    _same(_input(name))


@pytest.mark.parametrize("extra", [(), ("--passes", "2"), ("--passes", "3"), ("--lf-frame",), ("--hf-presets", "3"),
                                   ("--hf-presets", "5", "--passes", "2")])
def test_emulated_lanes_match_oracle_on_synthetic_frames(extra):
    # ragged right / bottom groups, 17 of the 27 transform types (DCT64 the largest), several groups per warp
    _same(bench.synth_frame(1000, 600, 7, extra=extra))


# tools/synth_enc.cc --all-types: every one of the 27 transform types, DCT128 .. DCT256 (128 to 1024 blocks, order ids
# 10-12) included, also in partial groups at the ragged edges; 2600 wide: on both sides of an LF-group boundary
ALL_TYPES_FRAMES = [((1000, 600), 7), ((2600, 700), 5)]


@pytest.mark.parametrize("extra", [(), ("--passes", "2"), ("--passes", "3"), ("--hf-presets", "5")],
                         ids=["staged", "passes2", "passes3", "presets5_general"])
@pytest.mark.parametrize("size,seed", ALL_TYPES_FRAMES)
def test_emulated_lanes_match_oracle_on_all_transform_types(size, seed, extra):
    # one HF preset: the staged variant (cluster maps and ANS tables in shared memory); five presets' cluster maps
    # (37 KB) exceed the staging budget and select the general variant
    _same(bench.synth_frame(size[0], size[1], seed, extra=("--all-types",) + extra))


@pytest.mark.parametrize("ttype", [19, 21, 22, 23, 24, 25, 26])
def test_emulated_lanes_match_oracle_on_one_transform_type(ttype):
    # a frame tiled with DCT64x32 or one of the six largest types wherever it fits (DCT8 elsewhere)
    _same(bench.synth_frame(1000, 600, 3, extra=("--only-type", str(ttype))))


def test_lane_records_hold_every_transform_type():
    """The transform-type records of the lanes decoder unpack to kTransformInfo for all 27 types (DCT256's 1024 blocks
    included), and its varblock record keeps type, context offset and position at their largest values."""
    L = oracle_lib.emu_lib()
    L.jxle_hf_record_check.restype = ctypes.c_int
    assert L.jxle_hf_record_check() == 0


def test_emulated_lanes_reject_truncated_streams():
    data = _input("opsin_inverse")
    for cut in (len(data) // 2, len(data) - 9):
        with pytest.raises(oracle_lib.OracleError) as e1:
            oracle_lib.OracleImage(data[:cut], threads=2)
        with pytest.raises(oracle_lib.OracleError) as e2:
            oracle_lib.OracleImage(data[:cut], threads=2, emu=True)
        assert e1.value.code == e2.value.code


@pytest.mark.parametrize("seed", range(8))
def test_device_bit_reader_matches_host_reader(seed):
    """DevBitReader (kernels/common.cuh) is shared by all three entropy kernels: random offsets / widths / peeks against
    host/bitreader.h, position included."""
    L = oracle_lib.emu_lib()
    L.jxle_bitreader_selftest.restype = ctypes.c_uint64
    L.jxle_bitreader_selftest.argtypes = [ctypes.c_uint64, ctypes.c_uint32]
    assert L.jxle_bitreader_selftest(seed, 12000) == 0


@pytest.mark.parametrize("seed", range(4))
def test_device_hybrid_uint_matches_closed_form(seed):
    L = oracle_lib.emu_lib()
    L.jxle_hybrid_uint_selftest.restype = ctypes.c_uint64
    L.jxle_hybrid_uint_selftest.argtypes = [ctypes.c_uint64, ctypes.c_uint32]
    assert L.jxle_hybrid_uint_selftest(seed, 20000) == 0
