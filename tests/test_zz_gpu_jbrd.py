"""JPEG bitstream reconstruction on the GPU (jxlb_reconstruct_jpeg: HF decode to the coefficients, then the scan
encoder kernels of kernels/jpeg.cu) against the oracle's scalar encoder and the reference's digests."""
import ctypes
import hashlib

import numpy as np
import pytest

from conftest import fixture_bytes

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]

JPEG_FIXTURES = ["cafe", "bench_oriented_brg", "grayscale_jpeg", "genshin_ycbcr_420", "issue_425"]


def test_brotli_library_loads():
    ctypes.CDLL("libbrotlidec.so.1").BrotliDecoderDecompress  # noqa: B018 - a missing library must fail, not skip


def test_reconstruct_matches_oracle_then_decoder_is_clean(oracle):
    import jbr_lib
    import jxl_oxide_b200 as J
    dec = J.Decoder(0)
    for name in JPEG_FIXTURES:
        data = fixture_bytes(name, "input.jxl")
        got = dec.reconstruct_jpeg(data)
        assert got == jbr_lib.reconstruct_jpeg(data), name
        assert hashlib.sha256(got).hexdigest() == fixture_bytes(name, "ref_jpeg_sha256.txt").decode().strip(), name
    # the same decoder then decodes a regular image bit-exactly: nothing of the reconstructions leaks into it
    data = fixture_bytes("bike", "input.jxl")
    dec.decode(data)
    got = dec.frame_planar(0)
    want, _, _ = oracle.OracleImage(data, threads=4).frame(0)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_jxl_image_api():
    import jxl_oxide_b200 as J
    data = fixture_bytes("issue_425", "input.jxl")
    img = J.JxlImage.read(data)
    assert img.jpeg_reconstruction_status() == 1 and J.jpeg_reconstruction_status(data) == 1
    assert img.reconstruct_jpeg() == fixture_bytes("issue_425", "ref.jpg")
    img.render_frame(0)  # the decoded frames stay available
    assert J.jpeg_reconstruction_status(fixture_bytes("bike", "input.jxl")) == 0


def test_no_jbrd_box_is_unavailable():
    import jxl_oxide_b200 as J
    with pytest.raises(J.JxlError) as e:
        J.Decoder(0).reconstruct_jpeg(fixture_bytes("bike", "input.jxl"))
    assert e.value.code == J.ERR_UNSUPPORTED and "unavailable" in str(e.value)


def test_allocation_budget():
    import jxl_oxide_b200 as J
    data = fixture_bytes("cafe", "input.jxl")
    small = J.Decoder(0, mem_limit=1 << 20)
    for _ in range(2):  # fails the same way twice: the failed call left nothing behind
        with pytest.raises(J.JxlError) as e:
            small.reconstruct_jpeg(data)
        assert e.value.code == J.ERR_OUT_OF_MEMORY
    assert hashlib.sha256(J.Decoder(0, mem_limit=1 << 30).reconstruct_jpeg(data)).hexdigest() == \
        fixture_bytes("cafe", "ref_jpeg_sha256.txt").decode().strip()


def test_launch_count_does_not_grow_with_image_size():
    """The scan encoder's launches per scan are fixed: cafe and genshin_ycbcr_420 (one scan each) cost the same."""
    import jxl_oxide_b200 as J
    counts = []
    for name in ("cafe", "genshin_ycbcr_420"):
        data = fixture_bytes(name, "input.jxl")
        dec = J.Decoder(0)
        c0 = dec.launch_count()
        # the same decode up to the coefficients, nothing copied out
        assert dec._L.jxlb_decode_hf_groups(dec._h, data, len(data), None, 0, None, None) == J.OK
        c1 = dec.launch_count()
        dec.reconstruct_jpeg(data)
        c2 = dec.launch_count()
        counts.append((c2 - c1) - (c1 - c0))
    assert counts[0] == counts[1] and 0 < counts[0] < 40, counts
