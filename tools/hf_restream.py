"""Builds and runs tools/hf_restream.cc: an existing VarDCT file with its HF passes rewritten with LZ77 codes (rle or
match) or in an entropy-code form of synth_enc's --code (prefix, ans-forms or configs), everything else kept. Test infrastructure; the binary goes to a per-user temporary directory keyed by its
sources, since the source tree may be read-only.

    python tools/hf_restream.py IN.jxl OUT.jxl rle|match|prefix|ans-forms|configs
"""
import glob
import hashlib
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "jxl_oxide_b200", "csrc", "host")
ORACLE = os.path.join(ROOT, "oracle")
SRCS = [os.path.join(ROOT, "tools", "hf_restream.cc")] + \
       [os.path.join(ORACLE, f) for f in ("oracle_capi.cc", "oracle_modular.cc", "oracle_vardct.cc", "oracle_render.cc")] + \
       [os.path.join(HOST, f) for f in ("entropy.cc", "headers.cc", "modular_syntax.cc", "frame_syntax.cc", "planner.cc", "icc.cc")]


def tool():
    """Path of the built restreamer (compiled on first use)."""
    deps = SRCS + [os.path.join(ROOT, "tools", "synth_enc.cc")] + sorted(glob.glob(os.path.join(HOST, "*.h")) +
                                                                       glob.glob(os.path.join(HOST, "*.inc")) +
                                                                       glob.glob(os.path.join(ORACLE, "*.h")))
    digest = hashlib.sha256()
    for p in deps:
        with open(p, "rb") as f:
            digest.update(f.read())
    d = os.path.join(tempfile.gettempdir(), f"jxlb_restream_{os.getuid()}", digest.hexdigest()[:16])
    os.makedirs(d, exist_ok=True)
    exe = os.path.join(d, "hf_restream")
    if not os.path.exists(exe):
        tmp = f"{exe}.{os.getpid()}"
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                               "-DJXLB_ENTROPY_TRACE", "-o", tmp] + SRCS)
        os.replace(tmp, exe)
    return exe


def restream(data: bytes, mode: str):
    """(restreamed file, values the decoder takes from LZ77 copies as the restreamer counted them); for the
    entropy-code forms, (restreamed file, the restreamer's stderr with its "code-form:" report)."""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.jxl"), os.path.join(d, "out.jxl")
        with open(src, "wb") as f:
            f.write(data)
        r = subprocess.run([tool(), src, dst, mode], capture_output=True, text=True, check=True)
        with open(dst, "rb") as f:
            out = f.read()
        if mode not in ("rle", "match"):
            return out, r.stderr
        return out, int(r.stderr.split("values copied")[0].split(":")[-1])


if __name__ == "__main__":
    if len(sys.argv) != 4:
        sys.exit(__doc__)
    with open(sys.argv[1], "rb") as f:
        out, n = restream(f.read(), sys.argv[3])
    with open(sys.argv[2], "wb") as f:
        f.write(out)
    print(f"{len(out)} bytes", f"{n} values copied" if sys.argv[3] in ("rle", "match") else n.strip())
