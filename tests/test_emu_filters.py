"""Host emulation of the column-strip restoration-filter kernel (kernels/filter_strip.cuh).

The kernel's phase functions (Gaborish, EPF step-1 distance maps, step-1 weighted sums, step 2 + colour) are plain
functions of (thread id, shared window), and the per-pixel formulas they call (kernels/pixel_math.cuh) are those of every
filter kernel; tests/emu/ compiles them for the host, runs every CTA thread by thread and
phase by phase over the frame's interior and compares each pixel with the oracle's own Gaborish / EPF / XYB stages
(bit patterns). The device launch (TMA window load, barriers, border tiles in the general kernel) is covered by
tests/test_gpu_parity.py and tests/test_zz_gpu_pipeline.py on a GPU.
"""
import ctypes
import os

import numpy as np
import pytest

import bench
import oracle_lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _stats(reset=False):
    L = oracle_lib.emu_lib()
    out = (ctypes.c_uint64 * 3)()
    L.jxle_strip_stats(out, int(reset))
    return list(out)


def _check(data, min_pixels):
    _stats(reset=True)
    want = oracle_lib.OracleImage(data, threads=4)
    got = oracle_lib.OracleImage(data, threads=4, emu=True)
    frames, compared, differ = _stats()
    assert frames >= 1 and compared >= min_pixels, "the emulated strip filter did not run"
    assert differ == 0, f"{differ} of {compared} interior samples differ from the oracle's filter stages"
    for i in range(want.num_frames):
        a, b = want.frame(i)[0], got.frame(i)[0]
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"frame {i} differs"


@pytest.mark.parametrize("size,seed", [((1000, 600), 7), ((520, 392), 11), ((2000, 1500), 3), ((712, 520), 9)])
def test_strip_filter_matches_oracle_on_synthetic_frames(size, seed):
    # per-block sigma from the frame's quantisation field and sharpness map, all 8x8-block border cases, ragged last tiles
    _check(bench.synth_frame(size[0], size[1], seed), 3 * (size[0] - 100) * (size[1] - 100))


@pytest.mark.parametrize("size,seed", [((1000, 600), 7), ((2600, 700), 5)])
def test_strip_filter_matches_oracle_on_all_transform_types(size, seed):
    # tools/synth_enc.cc --all-types: EPF sigma over 64x64 .. 256x256 varblocks (one quantisation value per varblock)
    _check(bench.synth_frame(size[0], size[1], seed, extra=("--all-types",)), 3 * (size[0] - 100) * (size[1] - 100))


def test_strip_filter_single_epf_step():
    # epf_iters == 1: step 1 is the last step and writes through the colour stage
    _check(bench.synth_frame(520, 392, 11, extra=("--epf-iters", "1")), 3 * 400 * 280)


@pytest.mark.parametrize("name", ["benchmark-data/starrail.d1-e6.jxl", "opsin_inverse/input.jxl", "minecraft_vardct_e7/input.jxl",
                                  "noise/input.jxl"])
def test_strip_filter_matches_oracle_on_libjxl_frames(name):
    # libjxl's own d1 frames: Gaborish + one EPF step; `noise` leaves the colour stage to a later kernel
    with open(os.path.join(GOLDEN, name), "rb") as f:
        _check(f.read(), 3 * 400 * 500)


def test_filter_launch_geometry():
    """The strip kernel's rectangle + the general kernel's 1-D border grid tile every frame size exactly once; strip windows stay
    inside the image and start on 16-byte boundaries (TMA) whenever the width is a multiple of four."""
    L = oracle_lib.emu_lib()
    L.jxle_filter_geometry_check.restype = ctypes.c_int
    sizes = [(128, 96), (129, 97), (160, 128), (500, 606), (520, 392), (1000, 600), (1001, 601), (2560, 1440), (3840, 2160), (7680, 4320),
             (7681, 4319), (4096, 97), (131, 4000)]
    sizes += [(w, h) for w in range(120, 330, 7) for h in (96, 100, 127, 128, 131, 161)]
    for w, h in sizes:
        assert L.jxle_filter_geometry_check(w, h) == 0, (w, h)
