"""Every entropy-code form the decoder reads, on streams whose decoded values are known (tests/entropy_forms_lib.py).

tools/synth_enc.cc --code writes all codes of a frame as prefix codes (simple and complex, codes longer than the
10-bit root table), as ANS with each histogram form (single symbol, two symbols, flat, general at shifts 0..13, RLE)
at log alphabet 6-8, with a hybrid-uint config per cluster, or with 65-256 clusters (complex cluster maps with and
without move-to-front, simple maps with nbits 0..3). The writer builds its own alias tables and prefix codes and checks
the product's parser against them, so an error in host/entropy.cc shared by the oracle and the device still fails
here. The oracle must decode each stream to the image it was made from (--dump-raw) or to what the same frame decodes
to in the default code; the host emulations of the device's Modular and HF stream code must match the oracle; and each
form must reach the branches it is written for, as the writer reports them."""
import ctypes

import numpy as np
import pytest

import entropy_forms_lib as ef
import oracle_lib
from test_emu_modular import _same as modular_emu_same
from test_emu_modular import emu  # noqa: F401  (the Modular stream emulation fixture)

MOD_IDS = [c[0] for c in ef.MODULAR]
VAR_IDS = [c[0] for c in ef.VARDCT]


def _frames_equal(a, b):
    assert a.num_frames == b.num_frames
    for i in range(a.num_frames):
        x, y = a.frame(i)[0], b.frame(i)[0]
        assert x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"frame {i} differs"


@pytest.mark.parametrize("form", ef.MODULAR_FORMS)
@pytest.mark.parametrize("case", ef.MODULAR, ids=MOD_IDS)
def test_modular_form_decodes_to_the_image(oracle, case, form):
    data, ref, src, _ = ef.modular_case(case, form)
    got = oracle.OracleImage(data, threads=4)
    if src is not None:
        assert np.array_equal(got.frame(0)[0], src.astype(np.float32) / np.float32(255))
    else:
        _frames_equal(oracle.OracleImage(ref, threads=4), got)


@pytest.mark.parametrize("form", ef.MODULAR_FORMS)
@pytest.mark.parametrize("case", ef.MODULAR, ids=MOD_IDS)
def test_modular_form_emulated_stream_code_matches_oracle(emu, case, form):  # noqa: F811
    modular_emu_same(emu, ef.modular_case(case, form)[0])


def _same_hf(want, got):
    wc, gc = want.stage("hf_coeff", np.int32), got.stage("hf_coeff", np.int32)
    assert len(wc) == len(gc) > 0
    for w, g in zip(wc, gc):
        assert w.shape == g.shape and np.array_equal(w, g), "HF coefficients differ"
    _frames_equal(want, got)


@pytest.mark.parametrize("form", ef.FORMS)
@pytest.mark.parametrize("case", ef.VARDCT, ids=VAR_IDS)
def test_vardct_form_decodes_like_the_default_code(oracle, case, form):
    data, ref, _ = ef.vardct_case(case, form)
    assert data != ref
    _same_hf(oracle.OracleImage(ref, threads=8, capture=True), oracle.OracleImage(data, threads=8, capture=True))


@pytest.mark.parametrize("form", ef.RESTREAM_FORMS)
@pytest.mark.parametrize("name", ef.REAL)
def test_restreamed_fixture_decodes_like_the_original(oracle, name, form):
    data, _ = ef.restreamed(name, form)
    assert data != ef.golden(name)
    _same_hf(oracle.OracleImage(ef.golden(name), threads=8, capture=True), oracle.OracleImage(data, threads=8, capture=True))


def _hf_streams():
    L = oracle_lib.emu_lib()
    L.jxle_hf_streams.restype = ctypes.c_uint64
    return L.jxle_hf_streams()


def _vardct_inputs():
    out = [pytest.param(("synth", c, f), id=f"{c[0]}-{f}") for c in ef.VARDCT for f in ef.FORMS]
    return out + [pytest.param(("real", n, f), id=f"{n}-{f}") for n in ef.REAL for f in ef.RESTREAM_FORMS]


def vardct_input(spec):
    kind, what, form = spec
    return ef.vardct_case(what, form)[0] if kind == "synth" else ef.restreamed(what, form)[0]


@pytest.mark.parametrize("spec", _vardct_inputs())
def test_vardct_form_emulated_hf_lanes_match_oracle(spec):
    data = vardct_input(spec)
    before = _hf_streams()
    want = oracle_lib.OracleImage(data, threads=4, capture=True)
    got = oracle_lib.OracleImage(data, threads=4, capture=True, emu=True)
    assert _hf_streams() > before, "the emulated HF path did not run"
    _same_hf(want, got)


# ---- each form reaches the branches it targets (the writer's report, summed over every input of the form) ----

def _union(form):
    reps = ef.all_reports(form)
    tot = {}
    for r in reps:
        assert r["codes"] > 0
        for k, v in r.items():
            if k in ("shifts", "log_alphas", "map_nbits", "map_mtf", "configs"):
                tot[k] = tot.get(k, 0) | v
            elif k.startswith("max_") or k == "root_bits":
                tot[k] = max(tot.get(k, 0), v)
            elif isinstance(v, list):
                tot[k] = [a + b for a, b in zip(tot.get(k, [0] * len(v)), v)]
            else:
                tot[k] = tot.get(k, 0) + v
    return reps, tot


def test_prefix_form_reaches_every_prefix_branch():
    reps, t = _union("prefix")
    for r in reps:  # every code of every input is a prefix code, and each has a code past the root table
        assert r["prefix_codes"] == r["codes"] and r["max_prefix_len"] == 15 > r["root_bits"] and r["long_codes"] > 0
    assert all(n > 0 for n in t["nsym"]), t["nsym"]  # simple codes of 1, 2, 3 and 4 symbols
    assert all(n > 0 for n in t["tree_select"])
    assert t["hskip0"] > 0 and t["hskip2"] > 0 and t["hskip3"] > 0
    assert t["repeat16"] > 0 and t["repeat17"] > 0
    assert t["single_symbol"] > 0


def test_ans_forms_reach_every_histogram_form():
    reps, t = _union("ans-forms")
    assert all(r["prefix_codes"] == 0 for r in reps)
    for k in ("ans_unary", "ans_binary", "ans_flat", "ans_general", "ans_rle"):
        assert t[k] > 0, k
    assert t["shifts"] == (1 << 14) - 1, hex(t["shifts"])  # every shift 0..13
    assert t["log_alphas"] == 0b111 << 6, hex(t["log_alphas"])  # log alphabet 6, 7 and 8


def test_configs_form_covers_the_config_space():
    from_writer = [(0, 0, 0), (1, 0, 1), (2, 1, 1), (3, 0, 3), (4, 2, 2), (5, 1, 3), (6, 3, 3), (7, 0, 7), (8, 0, 0),
                   (1, 1, 0), (4, 2, 0), (5, 0, 0), (3, 1, 0), (6, 0, 1)]  # kFormConfigs of tools/synth_enc.cc
    _, t = _union("configs")
    used = [c for i, c in enumerate(from_writer) if t["configs"] >> i & 1]
    assert {c[0] for c in used} == set(range(9))  # split_exponent 0 .. log alphabet size
    assert any(c[1] + c[2] == c[0] > 0 for c in used) and any(c[2] > 0 for c in used)


def test_clusters_form_reaches_large_cluster_counts():
    _, t = _union("clusters")
    assert t["max_clusters"] == 256
    assert t["max_ans_table_bytes"] > ef.hf_ans_smem_bytes()  # ANS tables read from global memory on the device
    assert t["map_mtf"] == 0b11  # complex maps with and without move-to-front
    assert t["map_nbits"] == 0b1111  # simple maps with nbits 0..3


def test_lz77_form_reaches_every_lz77_branch():
    reps = ef.all_reports("lz77")
    assert {r["length_sel"] for r in reps} == {0, 1, 2, 3}  # min_length 3, 4, 5 + u(2), 9 + u(8)
    assert {r["symbol_sel"] for r in reps} == {0, 3}  # min_symbol 224 and 8 + u(15); 512 and 4096 exceed ANS alphabets
    assert sum(r["copies_values"] > 0 for r in reps) >= len(reps) - 1
    assert sum(r["far"] for r in reps) > 0 and sum(r["cross_channel"] for r in reps) > 0  # copies across channels
    assert sum(r["special"] for r in reps) > 0  # "dy rows up, dx over": multiplier * dy + dx
    assert sum(r["from_start"] for r in reps) > 0  # distances the decoder clamps to the values decoded so far
    assert sum(r["past_window"] for r in reps) > 0  # copies after 2^20 values: the window has wrapped


# ---- streams the decoder must reject (the oracle shares host/entropy.cc: the writer knows what it made invalid) ----

@pytest.mark.parametrize("name,flags", ef.REJECTED, ids=[r[0] for r in ef.REJECTED])
def test_rejected_stream_is_an_error(oracle, name, flags):
    data, err = ef.rejected(flags)
    if "oversub" in flags[-1] or flags[-1] == "ans-sum":  # host parse errors: the reference's own rule, checked here
        assert ef.parse_report(err)["rejected_by_parser"] == 1
    with pytest.raises(oracle.OracleError) as e:
        oracle.OracleImage(data, threads=2)
    # a stream cut short by the end of its section is truncated input (3) to the host
    assert e.value.code in ((1, 3) if flags[-1] == "truncate" else (1,))
    if flags[-1] == "ans-state":
        assert "final state" in str(e.value)
