"""The synthetic Modular lossless stream (tools/synth_enc.cc --modular: YCoCg RCT + default Squeeze + weighted predictor,
BASELINE config #4) decodes, through the oracle, to exactly the image it was made from: the encoder's forward transforms
are inverted bit for bit by the restated reference path (and the stream's syntax is what the shared parser expects)."""
import subprocess

import numpy as np
import pytest

import bench


@pytest.mark.parametrize("w,h,seed", [(600, 400, 3), (1100, 700, 5), (513, 900, 2)])
def test_lossless_round_trip(oracle, tmp_path, w, h, seed):
    tool = bench.synth_tool()
    jxl, raw = str(tmp_path / "m.jxl"), str(tmp_path / "m.raw")
    subprocess.check_call([tool, "--modular", "--width", str(w), "--height", str(h), "--seed", str(seed), "-o", jxl, "--dump-raw", raw],
                          stderr=subprocess.DEVNULL)
    img = oracle.OracleImage(open(jxl, "rb").read(), threads=4)
    got = img.frame(0)[0]
    img.close()
    src = np.fromfile(raw, dtype=np.int32).reshape(3, h, w)
    assert got.shape == src.shape
    assert np.array_equal(got, src.astype(np.float32) / np.float32(255)), "the stream is not lossless"
