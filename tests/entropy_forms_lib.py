"""Streams in every entropy-code form of tools/synth_enc.cc --code (prefix, ans-forms, configs, clusters), and the real
VarDCT fixtures with their HF passes rewritten in a form by tools/hf_restream.cc, each with its ground truth and the
writer's report of the branches its codes reach. Shared by tests/test_entropy_forms.py (oracle and host emulation) and
tests/test_zz_gpu_entropy_forms.py (device). Test infrastructure only."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import hf_restream  # noqa: E402

FORMS = ["prefix", "ans-forms", "configs", "clusters"]
MODULAR_FORMS = FORMS + ["lz77"]  # LZ77 with special distances scaled by the widest channel: Modular streams only
RESTREAM_FORMS = ["prefix", "ans-forms", "configs"]  # clusters needs the contexts, which the restreamer does not see

# (id, width, height, seed, flags): partial edge groups, a YCbCr 4:2:0 and an extra-channel frame (coded without
# transforms), and the RCT + Squeeze frame
MODULAR = [("1100x700", 1100, 700, 5, []), ("513x900", 513, 900, 2, []),
           ("ycbcr420", 300, 200, 3, ["--ycbcr", "420"]),
           ("extra", 520, 300, 4, ["--extra", "alpha:8:0:1", "--extra", "spot:12:1:1"]),
           # one group of 3 colour and 14 extra channels: one stream of 1.1 M values, past the 2^20-value LZ77 window
           ("17ch_256x256", 256, 256, 6, ["--extra", "unknown:8:0:1"] * 14)]
VARDCT = [("passes3_presets3", 600, 500, 3, ["--passes", "3", "--hf-presets", "3"]),
          ("ycbcr420", 1000, 600, 7, ["--ycbcr", "420"])]
REAL = ["cafe", "genshin_ycbcr_420"]

_DIR = tempfile.mkdtemp(prefix="jxlb_entropy_forms_")
_CACHE = {}


def parse_report(text):
    out = {}
    m = re.search(r"lz77-modular: (.*)", text)
    if m:  # --code lz77
        text = "code-form: " + m.group(1)
    m = re.search(r"code-form: (.*)", text)
    assert m, text
    for kv in m.group(1).split():
        k, v = kv.split("=")
        out[k] = [int(x, 0) for x in v.split(",")] if "," in v else int(v, 0)
    return out


def synth(w, h, seed, flags, form=None, raw=False):
    """(bytes, report or None, raw int32 samples or None) of one synth_enc frame."""
    key = (w, h, seed, tuple(flags), form, raw)
    if key not in _CACHE:
        path = os.path.join(_DIR, f"{len(_CACHE)}.jxl")
        args = [bench.synth_tool(), "--width", str(w), "--height", str(h), "--seed", str(seed), "-o", path] + flags
        if form:
            args += ["--code", form]
        if raw:
            args += ["--dump-raw", path + ".raw"]
        r = subprocess.run(args, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        src = np.fromfile(path + ".raw", dtype=np.int32).reshape(3, h, w) if raw else None
        with open(path, "rb") as f:
            _CACHE[key] = (f.read(), parse_report(r.stderr) if form else None, src)
    return _CACHE[key]


def golden(name):
    with open(os.path.join(ROOT, "tests", "golden", name, "input.jxl"), "rb") as f:
        return f.read()


def restreamed(name, form):
    key = ("restream", name, form)
    if key not in _CACHE:
        data, err = hf_restream.restream(golden(name), form)
        _CACHE[key] = (data, parse_report(err), None)
    return _CACHE[key][:2]


def modular_case(case, form):
    """(coded bytes, reference bytes or None, raw samples or None, report)."""
    _, w, h, seed, flags = case
    flags = ["--modular"] + flags
    if len(flags) == 1:  # RCT + Squeeze: --dump-raw holds the image
        data, rep, src = synth(w, h, seed, flags, form, raw=True)
        return data, None, src, rep
    data, rep, _ = synth(w, h, seed, flags, form)
    return data, synth(w, h, seed, flags)[0], None, rep


def vardct_case(case, form):
    """(coded bytes, the same frame in the default code, report)."""
    _, w, h, seed, flags = case
    data, rep, _ = synth(w, h, seed, flags, form)
    return data, synth(w, h, seed, flags)[0], rep


def all_reports(form):
    reps = [modular_case(c, form)[3] for c in MODULAR]
    if form == "lz77":
        return reps
    reps += [vardct_case(c, form)[2] for c in VARDCT]
    if form in RESTREAM_FORMS:
        reps += [restreamed(n, form)[1] for n in REAL]
    return reps


# (id, synth_enc flags) of streams the decoder must reject; see --corrupt in tools/synth_enc.cc
_M = ["--modular", "--width", "600", "--height", "400", "--seed", "3"]
_V = ["--width", "600", "--height", "400", "--seed", "3"]
REJECTED = [("ans_state_modular_group", _M + ["--corrupt", "ans-state"]),
            ("ans_state_hf_group", _V + ["--corrupt", "ans-state"]),
            ("prefix_stream_cut_short", _M + ["--code", "prefix", "--corrupt", "truncate"]),
            ("prefix_code_length_code_oversubscribed", _M + ["--code", "prefix", "--corrupt", "oversub-clcl"]),
            ("prefix_lengths_oversubscribed", _M + ["--code", "prefix", "--corrupt", "oversub-lengths"]),
            ("ans_counts_past_4096", _V + ["--code", "ans-forms", "--corrupt", "ans-sum"])]


def rejected(flags):
    """(bytes, writer stderr) of an invalid stream."""
    key = ("rejected", tuple(flags))
    if key not in _CACHE:
        path = os.path.join(_DIR, f"{len(_CACHE)}.jxl")
        r = subprocess.run([bench.synth_tool(), "-o", path] + flags, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        with open(path, "rb") as f:
            _CACHE[key] = (f.read(), r.stderr)
    return _CACHE[key]


def hf_ans_smem_bytes():
    """kHfAnsSmemBytes of kernels/kernels.h: the largest HF ANS table set the device stages in shared memory."""
    with open(os.path.join(ROOT, "jxl_oxide_b200", "csrc", "kernels", "kernels.h")) as f:
        m = re.search(r"kHfAnsSmemBytes = ([0-9* ]+);", f.read())
    return eval(m.group(1))  # noqa: S307  (a product of integer literals)
