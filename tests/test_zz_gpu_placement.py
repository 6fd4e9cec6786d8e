"""GPU tests of the varblock placement inside the HfMetadata stream kernel (kernels/placement.cuh).

A pipeline frame places its varblocks in the LF batch its HfMetadata streams ride, so a VarDCT frame reaches the heavy
stage without a CUDA stream: host:slot_before_heavy (streams taken before begin_heavy_stage) stays 0, and the frames
equal a stand-alone decoder's. A corrupted layout still fails with JXLB_ERR_BITSTREAM on both paths."""
import ctypes

import numpy as np
import pytest

import bench
from conftest import fixture_bytes

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

BAD_LAYOUT = ["hf_varblock_across_group", "hfmul_non_positive"]


def _standalone(data):
    import jxl_oxide_b200 as J
    img = J.JxlImage.read(data)
    return img.render_frame(0).image_planar()


def test_pipeline_takes_no_slot_before_heavy_stage():
    import jxl_oxide_b200 as J
    datas = [bench.synth_frame(3840, 2160, s) for s in (1, 2, 3, 4)] + [fixture_bytes("minecraft_vardct_e7", "input.jxl")]
    want = [_standalone(d) for d in datas]
    pipe = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        decs = [pipe.decoder(i) for i in range(pipe.workers())]
        for d in decs:
            d._L.jxlb_set_profile(d._h, 3)  # host phases only
            d.profile_reset()
        for i, d in enumerate(datas):
            pipe.submit(data=d, mode=pipe.OUT_PLANAR_F32, tag=i)
        while pipe.in_flight:
            tag, addr, nbytes = pipe.wait(want_output=True)
            w = want[tag]
            assert nbytes == w.nbytes
            got = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(addr), np.uint32).copy()
            pipe.release_output(addr)
            assert np.array_equal(got, w.reshape(-1).view(np.uint32)), f"frame {tag} differs from a stand-alone decoder's"
        early = sum(d.profile("host:slot_before_heavy")[0] for d in decs)
        holds = sum(d.profile("host:slot_hold")[0] for d in decs)
        waits = sum(d.profile("host:slot_wait")[0] for d in decs)
    finally:
        pipe.close()
    assert early == 0, f"{early} frames took their heavy slot before begin_heavy_stage()"
    assert holds == len(datas) and waits == len(datas)


@pytest.mark.parametrize("name", BAD_LAYOUT)
def test_bad_layout_is_a_bitstream_error(name):
    import jxl_oxide_b200 as J
    data = fixture_bytes("fuzz_findings", f"{name}.fuzz")
    dec = J.Decoder(0)
    with pytest.raises(J.JxlError) as e:
        dec.decode(data)
    assert e.value.code == J.ERR_BITSTREAM, str(e.value)
    pipe = J.Pipeline(0, workers=2, heavy_frames=1)
    try:
        pipe.submit(data=data)
        with pytest.raises(J.JxlError) as e:
            pipe.wait()
        assert e.value.code == J.ERR_BITSTREAM, str(e.value)
    finally:
        pipe.close()
