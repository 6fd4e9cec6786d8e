"""Host emulation of the warp-parallel varblock placement (kernels/placement.cuh) against the oracle's serial scan.

tests/emu/placement_emu.cc compiles the placement's per-lane steps for the host and runs them for 32 lanes, one step at
a time. Every LF group is placed twice, by the emulation and by the oracle (OracleBackend::build_block_info), and the
two must agree on the status and, for a valid layout, on blk_type, blk_mul and epf_sigma bit for bit:
  * the LF groups of every VarDCT fixture, of the bench frames (synth8k seeds 1-4) and of synth_enc --all-types frames;
  * seeded random tilings of a 256 x 256-cell LF group, and seeded corruptions of them: overlaps, gaps, out-of-range
    dct_select / hf_mul, a varblock across a 32-cell boundary, too few and too many records, a bad EPF sharpness.
The random tilings have tall varblocks next to short ones, so a placement that ignored the cells occupied by earlier
rows would disagree. The device kernels run the same code; tests/test_zz_gpu_placement.py covers them on the GPU.
"""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest

import bench
import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
GOLDEN = os.path.join(ROOT, "tests", "golden")
SRCS = ["placement_emu.cc", "launch_tables_host.cc"] + [os.path.join("..", "..", "oracle", f) for f in
                             ("oracle_capi.cc", "oracle_modular.cc", "oracle_vardct.cc", "oracle_render.cc")] + \
       [os.path.join("..", "..", "jxl_oxide_b200", "csrc", "host", f) for f in
        ("entropy.cc", "headers.cc", "modular_syntax.cc", "frame_syntax.cc", "planner.cc", "icc.cc")]
# (w8, h8) of each transform type in 8x8 cells, in type-id order
SIZES = [(1, 1), (1, 1), (1, 1), (1, 1), (2, 2), (4, 4), (1, 2), (2, 1), (1, 4), (4, 1), (2, 4), (4, 2), (1, 1), (1, 1),
         (1, 1), (1, 1), (1, 1), (1, 1), (8, 8), (4, 8), (8, 4), (16, 16), (8, 16), (16, 8), (32, 32), (16, 32), (32, 16)]
I32P = ctypes.POINTER(ctypes.c_int32)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("placement_emu") / "libjxlplaceemu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                           "-I/usr/local/cuda/include", "-DJXLO_BACKEND_FACTORY=make_placement_emu_backend", "-shared",
                           "-Wl,-Bsymbolic", "-o", out] + SRCS, cwd=EMU)
    L = oracle_lib._load(out, None)
    L.jxlpe_stats.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]
    L.jxlpe_stop_after_placement.argtypes = [ctypes.c_int]
    L.jxlpe_place.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, I32P, I32P, ctypes.c_int,
                              I32P, I32P, ctypes.POINTER(ctypes.c_float)]
    return L


def _stats(L):
    v = (ctypes.c_uint64 * 3)()
    L.jxlpe_stats(v, 1)
    return list(v)


def _frame_groups(L, data):
    """Places the LF groups of the first frame with HfMetadata both ways; returns (groups, invalid, mismatches)."""
    _stats(L)
    saved = oracle_lib._EMU_LIB
    oracle_lib._EMU_LIB = L
    L.jxlpe_stop_after_placement(1)
    try:
        oracle_lib.OracleImage(data, threads=4, emu=True)
    except oracle_lib.OracleError:
        pass  # stopped after the placement, or a fixture that fails elsewhere
    finally:
        L.jxlpe_stop_after_placement(0)
        oracle_lib._EMU_LIB = saved
    return _stats(L)


def _fixtures():
    files = sorted(glob.glob(os.path.join(GOLDEN, "*", "input.jxl")) + glob.glob(os.path.join(GOLDEN, "benchmark-data", "*.jxl")) +
                   glob.glob(os.path.join(GOLDEN, "fuzz_findings", "*.fuzz")))
    return [os.path.relpath(f, GOLDEN) for f in files]


def test_fixtures(emu):
    groups = 0
    for rel in _fixtures():
        with open(os.path.join(GOLDEN, rel), "rb") as f:
            n, bad, mismatch = _frame_groups(emu, f.read())
        assert mismatch == 0, f"{rel}: the emulated placement differs from the oracle's in {mismatch} of {n} LF groups"
        groups += n
    assert groups >= 10, "too few VarDCT LF groups among the fixtures"


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_bench_frames(emu, seed):
    n, bad, mismatch = _frame_groups(emu, bench.synth_frame(7680, 4320, seed))
    assert n == 12 and bad == 0 and mismatch == 0


@pytest.mark.parametrize("size,seed", [((1000, 600), 7), ((2600, 700), 5), ((2000, 1500), 3)])
def test_all_types_frames(emu, size, seed):
    n, bad, mismatch = _frame_groups(emu, bench.synth_frame(size[0], size[1], seed, extra=("--all-types",)))
    assert n >= 1 and bad == 0 and mismatch == 0


def _tiling(rng, bw=256, bh=256):
    """A random valid varblock list for a bw x bh group: types drawn per free cell in raster order, tall ones included."""
    occ = np.zeros((bh, bw), bool)
    sels = []
    for y in range(bh):
        for x in range(bw):
            if occ[y, x]:
                continue
            while True:
                t = int(rng.integers(0, 27)) if rng.random() < 0.5 else int(rng.choice([0, 4, 5, 6, 8, 10, 18, 19]))
                w, h = SIZES[t]
                if x % 32 + w <= 32 and y % 32 + h <= 32 and x + w <= bw and y + h <= bh and not occ[y:y + h, x:x + w].any():
                    break
            occ[y:y + h, x:x + w] = True
            sels.append(t)
    sels = np.array(sels, np.int32)
    muls = rng.integers(0, 12, len(sels)).astype(np.int32)  # hf_mul - 1
    return sels, muls


def _place(L, emu_flag, bw, bh, sels, muls, sharp, has_epf):
    raw = np.ascontiguousarray(np.stack([sels, muls]).astype(np.int32))
    sharp = np.ascontiguousarray(sharp, np.int32)
    out = [np.zeros((bh, bw), np.int32), np.zeros((bh, bw), np.int32), np.zeros((bh, bw), np.float32)]
    st = L.jxlpe_place(emu_flag, bw, bh, len(sels), raw.ctypes.data_as(I32P), sharp.ctypes.data_as(I32P), int(has_epf),
                       out[0].ctypes.data_as(I32P), out[1].ctypes.data_as(I32P),
                       out[2].ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    return st, out


def _same(L, sels, muls, bw=256, bh=256, sharp=None, has_epf=True):
    if sharp is None:
        sharp = np.zeros((bh, bw), np.int32)
    st_e, got = _place(L, 1, bw, bh, sels, muls, sharp, has_epf)
    st_o, want = _place(L, 0, bw, bh, sels, muls, sharp, has_epf)
    assert st_e == st_o, f"status: emulation {st_e}, oracle {st_o}"
    if st_o == 0:
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))
    return st_o


@pytest.mark.parametrize("seed", range(6))
def test_random_tilings(emu, seed):
    rng = np.random.default_rng(seed)
    sels, muls = _tiling(rng)
    sharp = rng.integers(0, 8, (256, 256)).astype(np.int32)
    assert _same(emu, sels, muls, sharp=sharp) == 0
    assert _same(emu, sels, muls, has_epf=False) == 0
    # ragged groups at a frame's right / bottom edge
    bw, bh = 256 - int(rng.integers(1, 40)), 256 - int(rng.integers(1, 40))
    sels2, muls2 = _tiling(rng, bw, bh)
    assert _same(emu, sels2, muls2, bw, bh) == 0


def _corruptions(rng, sels, muls):
    """(name, sels, muls) variants of a valid list."""
    n = len(sels)
    out = []
    for _ in range(3):
        i = int(rng.integers(0, n))
        s = sels.copy()
        small = np.flatnonzero(np.isin(s, [0, 1, 2, 3, 6, 7]))
        j = int(rng.choice(small)) if len(small) else i
        s[j] = 5  # a 4x4 block where a small one was: overlaps what follows
        out.append(("overlap", s, muls))
        s = sels.copy()
        big = np.flatnonzero(np.isin(s, [4, 5, 10, 11, 18, 19, 20]))
        if len(big):
            s[int(rng.choice(big))] = 0  # an 8x8 block where a larger one was: a gap
            out.append(("gap", s, muls))
        s = sels.copy()
        s[i] = int(rng.choice([27, 40, -1]))
        out.append(("sel", s, muls))
        m = muls.copy()
        m[i] = int(rng.choice([-1, -7]))
        out.append(("hf_mul", sels, m))
        s = sels.copy()
        s[i] = int(rng.choice([18, 21, 24]))  # 8x8 .. 32x32 cells: crosses a 32-cell boundary unless aligned
        out.append(("boundary", s, muls))
        k = int(rng.integers(1, 20))
        out.append(("too_few", sels[:n - k], muls[:n - k]))
        extra = rng.integers(-3, 30, k).astype(np.int32)
        out.append(("too_many", np.concatenate([sels, extra]), np.concatenate([muls, extra])))
    return out


@pytest.mark.parametrize("seed", range(4))
def test_corrupted_tilings(emu, seed):
    rng = np.random.default_rng(100 + seed)
    sels, muls = _tiling(rng)
    seen = {}
    for name, s, m in _corruptions(rng, sels, muls):
        st = _same(emu, s, m)
        seen.setdefault(name, set()).add(st)
    for name in ("overlap", "sel", "hf_mul", "too_few"):
        assert seen[name] == {1}, f"{name}: a corrupted list was accepted"
    assert seen["too_many"] == {0}, "records after a full group must be ignored"
    sharp = np.zeros((256, 256), np.int32)
    sharp[int(rng.integers(0, 256)), int(rng.integers(0, 256))] = 9
    assert _same(emu, sels, muls, sharp=sharp) == 1
    assert _same(emu, sels, muls, sharp=sharp, has_epf=False) == 0


def test_row_fill_respects_occupied_cells(emu):
    """A tall block followed by 1x1 blocks: the second row must skip the tall block's cells."""
    bw, bh = 8, 2
    # row 0: a 1x2 (type 6: w=1, h=2) then seven 1x1; row 1: seven 1x1 right of the tall block
    sels = np.array([6] + [0] * 7 + [0] * 7, np.int32)
    muls = np.zeros(len(sels), np.int32)
    assert _same(emu, sels, muls, bw, bh) == 0
    st, out = _place(emu, 1, bw, bh, sels, muls, np.zeros((bh, bw), np.int32), False)
    assert st == 0 and out[0][1, 0] == -(1 + 32) and (out[0][1, 1:] == 0).all()
