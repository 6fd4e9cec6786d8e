"""JPEG bitstream reconstruction without a GPU: the oracle's scalar scan encoder (oracle/oracle_jbr.cc) against the
reference's digests, the host build of the device scan encoder (tests/emu/jpeg_emu.cc) against the oracle, and the
reconstruction status / error paths of the shared host code (csrc/host/jbrd.cc)."""
import ctypes
import hashlib
import struct

import pytest

from conftest import fixture_bytes


@pytest.fixture(scope="module")
def jbr():
    import jbr_lib
    jbr_lib.build()
    return jbr_lib

JPEG_FIXTURES = ["cafe", "bench_oriented_brg", "grayscale_jpeg", "genshin_ycbcr_420", "issue_425"]


def boxes(data):
    """[(type, payload)] of an ISOBMFF JPEG XL container (32-bit box sizes, as in the fixtures)."""
    out, pos = [], 0
    while pos < len(data):
        size, = struct.unpack(">I", data[pos:pos + 4])
        size = size or len(data) - pos
        out.append((data[pos + 4:pos + 8], data[pos + 8:pos + size]))
        pos += size
    return out


def container(bxs):
    return b"".join(struct.pack(">I", 8 + len(p)) + t + p for t, p in bxs)


def with_jbrd(data, payload):
    return container([(t, payload if t == b"jbrd" else p) for t, p in boxes(data)])


def brotli_uncompressed(raw):
    """A Brotli stream holding `raw` in one uncompressed meta-block (RFC 7932 9.1-9.2), then an empty last one."""
    assert 0 < len(raw) <= 1 << 16
    header = ((len(raw) - 1) << 4) | (1 << 20)  # WBITS 16, ISLAST 0, MNIBBLES 4, MLEN - 1, ISUNCOMPRESSED
    return header.to_bytes(3, "little") + raw + b"\x03"


def data_section(jbrd, jpeg):
    """(offset, decoded bytes) of the Brotli data section at the end of a jbrd payload: the first offset whose suffix
    decodes, to bytes that the original JPEG contains."""
    dec = ctypes.CDLL("libbrotlidec.so.1")
    dec.BrotliDecoderDecompress.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p]
    for k in range(len(jbrd)):
        out, n = ctypes.create_string_buffer(1 << 16), ctypes.c_size_t(1 << 16)
        if dec.BrotliDecoderDecompress(len(jbrd) - k, jbrd[k:], ctypes.byref(n), out) == 1 and n.value and out.raw[:n.value] in jpeg:
            return k, out.raw[:n.value]
    raise AssertionError("no data section found")


@pytest.mark.parametrize("name", JPEG_FIXTURES)
def test_oracle_reconstructs_reference_digest(jbr, name):
    jpeg = jbr.reconstruct_jpeg(fixture_bytes(name, "input.jxl"))
    assert jpeg[:2] == b"\xff\xd8"
    assert hashlib.sha256(jpeg).hexdigest() == fixture_bytes(name, "ref_jpeg_sha256.txt").decode().strip()


def test_issue_425_is_the_original_file(jbr):
    assert jbr.reconstruct_jpeg(fixture_bytes("issue_425", "input.jxl")) == fixture_bytes("issue_425", "ref.jpg")


@pytest.mark.parametrize("name", JPEG_FIXTURES)
def test_emulated_kernels_match_oracle(jbr, name):
    data = fixture_bytes(name, "input.jxl")
    assert jbr.reconstruct_jpeg(data, emu=True) == jbr.reconstruct_jpeg(data)


def test_reconstruction_status(jbr):
    for name in JPEG_FIXTURES:
        assert jbr.jpeg_reconstruction_status(fixture_bytes(name, "input.jxl")) == 1, name
    for name in ("bike", "grayscale"):
        assert jbr.jpeg_reconstruction_status(fixture_bytes(name, "input.jxl")) == 0, name
    with pytest.raises(jbr.JbrError) as e:
        jbr.reconstruct_jpeg(fixture_bytes("bike", "input.jxl"))
    assert e.value.code == 2 and "unavailable" in str(e.value)


@pytest.mark.parametrize("keep", [0, 1, 8, 40, 120])
def test_truncated_jbrd_box(jbr, keep):
    data = fixture_bytes("cafe", "input.jxl")
    jbrd = dict(boxes(data))[b"jbrd"]
    bad = with_jbrd(data, jbrd[:keep])
    assert jbr.jpeg_reconstruction_status(bad) == 2
    with pytest.raises(jbr.JbrError):
        jbr.reconstruct_jpeg(bad)


def test_data_section_of_wrong_length(jbr):
    data = fixture_bytes("cafe", "input.jxl")
    jbrd = dict(boxes(data))[b"jbrd"]
    at, raw = data_section(jbrd, jbr.reconstruct_jpeg(data))
    same = with_jbrd(data, jbrd[:at] + brotli_uncompressed(raw))  # the stream builder itself is sound
    assert jbr.reconstruct_jpeg(same) == jbr.reconstruct_jpeg(data)
    for wrong in (raw + b"\0", raw[:-1]):
        with pytest.raises(jbr.JbrError) as e:
            jbr.reconstruct_jpeg(with_jbrd(data, jbrd[:at] + brotli_uncompressed(wrong)))
        assert e.value.code == 1, str(e.value)
