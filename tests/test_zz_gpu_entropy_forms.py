"""Every entropy-code form on the device (tests/entropy_forms_lib.py): the Modular stream kernel and the HF coefficient
decoder under each HF schedule must decode the prefix, ans-forms, configs, clusters and (Modular) lz77 streams, and
the real fixtures restreamed in a form, to what the oracle decodes (pixels and HF coefficients bit for bit), and must
report each invalid stream of entropy_forms_lib.REJECTED as an error value and stay usable. The oracle itself is
pinned to the known images by tests/test_entropy_forms.py."""
import numpy as np
import pytest

import entropy_forms_lib as ef
from test_entropy_forms import _vardct_inputs, vardct_input
from test_zz_gpu_hf_lz77 import _as_array

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800, method="thread")]


@pytest.fixture(scope="module")
def dec():
    import jxl_oxide_b200
    d = jxl_oxide_b200.Decoder(0)
    yield d
    d.close()


@pytest.mark.parametrize("form", ef.MODULAR_FORMS)
@pytest.mark.parametrize("case", ef.MODULAR, ids=[c[0] for c in ef.MODULAR])
def test_modular_form_on_device(dec, oracle, case, form):
    data = ef.modular_case(case, form)[0]
    dec.decode(data)
    got = dec.frame_planar(0)
    want = oracle.OracleImage(data, threads=8).frame(0)[0]
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("spec", _vardct_inputs())
def test_vardct_form_on_device_under_each_hf_schedule(dec, oracle, spec):
    data = vardct_input(spec)
    img = oracle.OracleImage(data, threads=8, capture=True)
    want, wc = img.frame(0)[0], img.stage("hf_coeff", np.int32)
    for streams in (0, 8, 32, 64):
        dec.set_hf_streams_per_cta(streams)
        try:
            dec.set_capture(True)
            dec.decode(data)
            got, gc = dec.frame_planar(0), dec.stage("hf_coeff", np.int32)
        finally:
            dec.set_capture(False)
            dec.set_hf_streams_per_cta(0)
        assert len(gc) == len(wc) > 0
        for g, w in zip(gc, wc):
            assert np.array_equal(g, w), f"HF coefficients differ at {streams} streams per CTA"
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), streams


def test_forms_in_the_pipeline(oracle):
    """A Modular prefix-coded frame and a VarDCT frame with 65-256 clusters, beside default-coded frames."""
    import jxl_oxide_b200 as J
    datas = [ef.modular_case(ef.MODULAR[0], "prefix")[0], ef.vardct_case(ef.VARDCT[0], "clusters")[0],
             ef.vardct_case(ef.VARDCT[0], "clusters")[1], ef.restreamed("cafe", "ans-forms")[0]]
    want = []
    for d in datas:
        img = oracle.OracleImage(d, threads=16)
        want.append(img.frame(0)[0])
        img.close()
    p = J.Pipeline(0, workers=4, heavy_frames=2)
    try:
        for i, d in enumerate(datas):
            p.submit(data=d, mode=p.OUT_PLANAR_F32, tag=i)
        seen = set()
        while p.in_flight:
            tag, addr, nbytes = p.wait(want_output=True)
            w = want[tag]
            assert nbytes == w.nbytes
            got = _as_array(addr, nbytes, np.float32, w.shape)
            p.release_output(addr)
            assert np.array_equal(got.view(np.uint32), w.view(np.uint32)), f"frame {tag} differs from the oracle"
            seen.add(tag)
        assert seen == set(range(len(datas)))
    finally:
        p.close()


@pytest.mark.parametrize("name,flags", ef.REJECTED, ids=[r[0] for r in ef.REJECTED])
def test_rejected_stream_is_an_error_value(dec, oracle, name, flags):
    import jxl_oxide_b200 as J
    data, _ = ef.rejected(flags)
    for streams in (0, 64):
        dec.set_hf_streams_per_cta(streams)
        try:
            with pytest.raises(J.JxlError) as e:
                dec.decode(data)
        finally:
            dec.set_hf_streams_per_cta(0)
        # a stream that reads past the end of its section is truncated input (3), as the host says of it
        assert e.value.code in ((3,) if flags[-1] == "truncate" else (1, 6)), (e.value.code, str(e.value))
    good = ef.synth(600, 400, 3, ["--modular"])[0]  # the decoder stays usable
    dec.decode(good)
    want = oracle.OracleImage(good, threads=8).frame(0)[0]
    assert np.array_equal(dec.frame_planar(0).view(np.uint32), want.view(np.uint32))
