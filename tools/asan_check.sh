#!/bin/bash
# Host-side memory / UB check without a GPU: the planner, syntax parsers and ICC code (product sources under
# jxl_oxide_b200/csrc/host) built together with the CPU oracle under AddressSanitizer + UBSan, then fed every fixture,
# the reference's fuzz corpus and N random mutations (bit flips, truncations, overwrites) of every small fixture.
#   bash tools/asan_check.sh [mutations per file, default 20]
set -e
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
OUT=/tmp/jxlb_asan
mkdir -p "$OUT"
H="$ROOT/jxl_oxide_b200/csrc/host"
g++ -std=c++17 -O1 -g -fPIC -fsanitize=address,undefined -fno-omit-frame-pointer -ffp-contract=off -pthread -shared -w \
    -o "$OUT/libjxloracle_asan.so" "$ROOT"/oracle/oracle_{capi,modular,vardct,render}.cc \
    "$H"/{entropy,headers,modular_syntax,frame_syntax,planner,icc,frame_index,jbrd}.cc "$ROOT"/oracle/oracle_jbr.cc \
    "$ROOT"/tests/emu/keyframes_capi.cc -ldl
cat > "$OUT/run.py" <<PY
import sys, os, ctypes, glob, random
sys.path.insert(0, "$ROOT/tests"); sys.path.insert(0, "$ROOT")
import oracle_lib
L = oracle_lib._load("$OUT/libjxloracle_asan.so", None)
def dec(data):
    st = ctypes.c_int(0); err = ctypes.create_string_buffer(512)
    h = L.jxlo_decode(data, len(data), 0, 2, 0, ctypes.byref(st), err, 512)
    if h: L.jxlo_free(h)
files = [f for f in sorted(glob.glob("$ROOT/tests/golden/*/input.jxl")) + sorted(glob.glob("$ROOT/tests/golden/fuzz_findings/*")) if os.path.isfile(f)]
for f in files: dec(open(f, "rb").read())
rng = random.Random(1); n = 0
for f in files:
    if "fuzz" in f or os.path.getsize(f) >= 400000: continue
    d = open(f, "rb").read()
    for _ in range(int(sys.argv[1])):
        m = bytearray(d); k = rng.choice(["flip", "trunc", "over"])
        if k == "flip":
            for _ in range(rng.randint(1, 4)): m[rng.randrange(len(m))] ^= 1 << rng.randrange(8)
        elif k == "trunc": m = m[:rng.randrange(1, len(m))]
        else:
            p = rng.randrange(len(m))
            for i in range(p, min(len(m), p + rng.randint(1, 16))): m[i] = rng.randrange(256)
        dec(bytes(m)); n += 1
# the synthetic frame kinds (previews, frames saved before or after the colour transform), whole, cut at every 1/64 of
# their length and at every byte of their first 64 after the image header (the preview's frame header and TOC), through
# the decoder, the keyframe index and the jbrd reader (behind grayscale_jpeg's jbrd box in a container)
import struct, frame_kinds_lib
u32 = ctypes.POINTER(ctypes.c_uint32)
L.jxlk_segments.argtypes = [ctypes.c_char_p, ctypes.c_size_t, u32, u32, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
L.jxlo_jpeg_reconstruction_status.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
def box(t, b): return struct.pack(">I", 8 + len(b)) + t + b
jpeg = open("$ROOT/tests/golden/grayscale_jpeg/input.jxl", "rb").read()
at = jpeg.index(b"jbrd") - 4
jbrd = jpeg[at + 8:at + struct.unpack(">I", jpeg[at:at + 4])[0]]
sig = bytes([0, 0, 0, 0x0c]) + b"JXL " + bytes([0x0d, 0x0a, 0x87, 0x0a])
head = len(frame_kinds_lib.synth_anim.image_header(frame_kinds_lib.W, frame_kinds_lib.H, False, preview=frame_kinds_lib.PREVIEW).bytes())
first, count, err = (ctypes.c_uint32 * 64)(), (ctypes.c_uint32 * 64)(), ctypes.c_int()
for d in frame_kinds_lib.STREAMS.values():
    for cut in sorted(set(range(1, len(d), max(1, len(d) // 64))) | set(range(head, head + 64)) | {len(d)}):
        m = d[:cut]
        dec(m)
        L.jxlk_segments(m, len(m), first, count, 64, ctypes.byref(err))
        c = sig + box(b"jbrd", jbrd) + box(b"jxlc", m)
        L.jxlo_jpeg_reconstruction_status(c, len(c))
        n += 1
print("inputs:", len(files) + len(frame_kinds_lib.STREAMS), "mutations:", n)
PY
ASAN="$(gcc -print-file-name=libasan.so)"
STD="$(gcc -print-file-name=libstdc++.so.6)"
# libstdc++ is preloaded too: python does not link it, and ASan must find __cxa_throw when it initialises
LD_PRELOAD="$ASAN $STD" ASAN_OPTIONS=detect_leaks=0:halt_on_error=1:allocator_may_return_null=1 UBSAN_OPTIONS=print_stacktrace=0 \
    python "$OUT/run.py" "${1:-20}" 2>&1 | tail -20
