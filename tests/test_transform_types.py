"""All 27 VarDCT transform types, from DCT8 to DCT256, on the CPU.

tools/synth_enc.cc --all-types puts every type into each frame (the six largest, DCT128 .. DCT256, also into partial
groups at the ragged right / bottom edges and next to LF-group boundaries); --dump-blocks writes the layout, so the
tests know each varblock's type without a stage of the decoder. The oracle's inverse transforms are checked here
against a float64 reference built from first principles; the GPU kernels are compared with the oracle in
tests/test_zz_gpu_transforms.py and the host-compiled HF decoder in tests/test_emu_lanes.py.
"""
import math
import os
import subprocess

import numpy as np
import pytest

import bench

# (w8, h8): size of each transform type in 8x8 blocks, in type-id order (kTransformInfo)
SIZES = [(1, 1), (1, 1), (1, 1), (1, 1), (2, 2), (4, 4), (1, 2), (2, 1), (1, 4), (4, 1), (2, 4), (4, 2), (1, 1), (1, 1),
         (1, 1), (1, 1), (1, 1), (1, 1), (8, 8), (4, 8), (8, 4), (16, 16), (8, 16), (16, 8), (32, 32), (16, 32), (32, 16)]
HUGE = [21, 22, 23, 24, 25, 26]  # DCT128, DCT128x64, DCT64x128, DCT256, DCT256x128, DCT128x256
# Types whose inverse transform is a plain 2-D DCT of the block. Hornuss (1), DCT2 (2), DCT4 (3), DCT4x8 / DCT8x4
# (12, 13) and AFV (14-17) are covered only by bit equality of the GPU and the oracle, and by the libjxl renderings.
DCT_TYPES = [0, 4, 5, 6, 7, 8, 9, 10, 11, 18, 19, 20, 21, 22, 23, 24, 25, 26]
ALL_TYPES_FRAMES = [((1000, 600), 7), ((2600, 700), 5), ((2000, 1500), 3)]


def layout(w, h, seed, extra=("--all-types",)):
    """(frame bytes, blocks): blocks is an (n, 3) array of (x, y, type), positions in 8x8 cells."""
    data = bench.synth_frame(w, h, seed, extra=extra)
    tag = "".join(extra).replace("-", "")
    path = os.path.join(bench._synth_cache(), f"blocks_{w}x{h}_s{seed}{tag}.txt")
    if not os.path.exists(path):
        tmp = f"{path}.{os.getpid()}"
        subprocess.check_call([bench.synth_tool(), "--width", str(w), "--height", str(h), "--seed", str(seed), "--distance", "1.0",
                               "-o", f"{tmp}.jxl", "--dump-blocks", tmp] + list(extra), stderr=subprocess.DEVNULL)
        with open(f"{tmp}.jxl", "rb") as f:
            assert f.read() == data, "--dump-blocks changed the frame"
        os.remove(f"{tmp}.jxl")
        os.replace(tmp, path)
    return data, np.loadtxt(path, dtype=np.int64, ndmin=2).reshape(-1, 3)


@pytest.mark.parametrize("size,seed", ALL_TYPES_FRAMES)
def test_all_types_layout(size, seed):
    w, h = size
    _, blocks = layout(w, h, seed)
    assert sorted(set(blocks[:, 2].tolist())) == list(range(27))
    bw, bh = (w + 7) // 8, (h + 7) // 8
    cover = np.zeros((bh, bw), np.int32)
    for x, y, t in blocks:
        bx, by = SIZES[t]
        assert x // 32 == (x + bx - 1) // 32 and y // 32 == (y + by - 1) // 32, "a varblock crosses a group boundary"
        cover[y:y + by, x:x + bx] += 1
    assert (cover == 1).all(), "varblocks must tile the frame"
    huge = blocks[np.isin(blocks[:, 2], HUGE)]
    right = [x for x, y, t in huge if x // 32 == (bw - 1) // 32]
    bottom = [y for x, y, t in huge if y // 32 == (bh - 1) // 32]
    if bw % 32 >= 16:
        assert right, "no large varblock in the partial groups at the right edge"
    if bh % 32 >= 8:
        assert bottom, "no large varblock in the partial groups at the bottom edge"
    if bw > 256:  # both sides of the LF-group boundary at 2048 samples
        assert any(x // 32 == 7 for x, y, t in huge) and any(x // 32 == 8 for x, y, t in huge)


@pytest.mark.parametrize("ttype", [6, 19] + HUGE)
def test_only_type_tiles_every_group(ttype):
    w, h = 1000, 600
    _, blocks = layout(w, h, 3, extra=("--only-type", str(ttype)))
    bw, bh = (w + 7) // 8, (h + 7) // 8
    tw, th = SIZES[ttype]
    want = 0
    for gy in range(0, bh, 32):
        for gx in range(0, bw, 32):
            want += (min(32, bw - gx) // tw) * (min(32, bh - gy) // th)
    assert want > 0 and int((blocks[:, 2] == ttype).sum()) == want
    assert set(blocks[:, 2].tolist()) <= {0, ttype}


def _idct_matrix(n):
    """m[i, k] = alpha_k cos(pi (i + 1/2) k / n), alpha_0 = 1, alpha_k = sqrt(2): the inverse DCT the decoder applies
    (samples = m @ coefficients); its inverse is m.T / n."""
    m = np.cos(np.pi * (np.arange(n)[:, None] + 0.5) * np.arange(n)[None, :] / n)
    m[:, 1:] *= math.sqrt(2.0)
    return m


def _box_mean_gain(n):
    """Mean over an 8-sample run (one 8x8 block) of the 8n-point basis function k, divided by the n-point basis function
    k at that block: sin(pi k / 2n) / (8 sin(pi k / 16n)) (sum of eight equally spaced cosines), 1 for k = 0."""
    k = np.arange(1, n, dtype=np.float64)
    return np.r_[1.0, np.sin(np.pi * k / (2 * n)) / (8 * np.sin(np.pi * k / (16 * n)))]


@pytest.mark.parametrize("size,seed", ALL_TYPES_FRAMES[:2])
def test_inverse_transforms_against_float64(oracle, size, seed):
    """Dequantisation, then the inverse transform of every DCT-shaped varblock, in float64 from first principles,
    against the oracle's `idct` stage. Inputs: the dequantised coefficients (`hf_dequant` stage, chroma from luma applied)
    and the LF image (`lf` stage).

    Layout: coefficient (u, v) of a W x H varblock sits at column u, row v of the block's own W x H area (horizontal
    frequency along x), the lowest bw x bh of them (bw = W / 8, bh = H / 8) replaced by the LLF corner. The layout is pinned
    independently by the DCT16x8 / DCT8x16 blocks of the libjxl-rendered fixtures that the oracle reproduces.
    LLF: the LF image holds the 8x8 box means of the low-frequency part of the block. Box-averaging the 8n-point basis
    function k gives the n-point basis function k times _box_mean_gain(n)[k], so the LLF corner is the bw x bh DCT of
    the LF values divided by the gains along both axes.
    Bound: float32 roundoff of a transform with log2(W H) butterfly levels plus the LLF scaling, 2 units of 2^-24 per
    level relative to sum |alpha_u alpha_v C_uv| of the block (the measured worst case is about half)."""
    w, h = size
    data, blocks = layout(w, h, seed)
    img = oracle.OracleImage(data, threads=8, capture=True)
    lf = [p.astype(np.float64) for p in img.stage("lf")]
    deq = [p.astype(np.float64) for p in img.stage("hf_dequant")]
    got = [p.astype(np.float64) for p in img.stage("idct")]
    img.close()
    assert [p.shape for p in got] == [(8 * ((h + 7) // 8), 8 * ((w + 7) // 8))] * 3
    for t in DCT_TYPES:
        sel = blocks[blocks[:, 2] == t]
        assert len(sel), f"type {t} missing from the frame"
        bw, bh = SIZES[t]
        mw, mh = _idct_matrix(8 * bw), _idct_matrix(8 * bh)
        fw, fh = _idct_matrix(bw).T / bw, _idct_matrix(bh).T / bh  # forward bw- / bh-point DCT
        gain = np.outer(_box_mean_gain(bh), _box_mean_gain(bw))
        alpha = np.outer(np.r_[1.0, np.full(8 * bh - 1, math.sqrt(2.0))], np.r_[1.0, np.full(8 * bw - 1, math.sqrt(2.0))])
        levels = math.log2(64 * bw * bh) + 2
        for c in range(3):
            for x, y, _ in sel:
                coeff = deq[c][8 * y:8 * (y + bh), 8 * x:8 * (x + bw)].copy()
                coeff[:bh, :bw] = (fh @ lf[c][y:y + bh, x:x + bw] @ fw.T) / gain
                want = mh @ coeff @ mw.T
                bound = 2 * levels * 2.0 ** -24 * (alpha * np.abs(coeff)).sum()
                err = np.abs(got[c][8 * y:8 * (y + bh), 8 * x:8 * (x + bw)] - want).max()
                assert err <= bound, f"type {t} at ({x}, {y}) channel {c}: error {err:.3g} > {bound:.3g}"
