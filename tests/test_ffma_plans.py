"""Host-only checks of the "fp32_ffma" path's launcher and of its kernel tests (no GPU; the plan hook then assumes 132 SMs):

* ev_debug_conv1d_plan gives a variant of conv1d_tm_kernel for every convolution the engine runs at the corpus's batches, within
  the 96 KB shared-memory attribute, and rejects what ev_op_conv1d rejects;
* the variant is a function of (B, L, C_out) alone -- C_in, K and the dilation enter only through the A tile's row limit --, so the
  operator cases of tests/test_ffma_kernels_gpu.py stand for every layer that shares a C_out;
* those cases launch every (layer, variant) and every (layer, batch variant, batch-1 variant) pair the engine can produce;
* the "fp32_ffma" launch lists: no split-K reduce, the FFMA attention, a transpose only for a channels-first mel.
"""
import itertools

import pytest

import am_plans
import ffma_cases
import voc_plans

SMEM_ATTR = 96 * 1024


def _engine_layers():
    for B, lens, frames in ffma_cases.engine_workloads():
        shapes = [(B, max(lens), max(frames))] + [(1, n, f) for n, f in zip(lens, frames)]
        for b, T, F in shapes:
            for r in am_plans.am_layers(b, T, F, "fp32_ffma", 1):
                if isinstance(r, dict):
                    yield r["kind"], b, r["L"], r["Cin"], r["Cout"], r["K"], 1
            for r in voc_plans.ffma_layers(b, F):
                yield r["kind"], b, r["L"], r["Cin"], r["Cout"], r["K"], r["dil"]


def test_every_engine_layer_has_a_plan_within_the_smem_attribute(lib):
    n = 0
    for kind, B, L, Cin, Cout, K, dil in _engine_layers():
        p = am_plans.conv1d_plan(lib, B, L, Cin, Cout, K, dil)
        assert p is not None, (kind, B, L, Cin, Cout, K, dil, lib.ev_last_error())
        assert (p["TXN"], p["NV"], p["TM"]) in {(8, 1, 8), (16, 1, 4), (16, 1, 8), (16, 2, 8)}
        assert p["BM"] == 256 // p["TXN"] * p["TM"] and p["BN"] == p["TXN"] * 4 * p["NV"]
        assert p["rows_a"] == p["BM"] + (K - 1) * dil <= 384 and p["a_ld"] % 8 == 2 and p["a_ld"] >= p["rows_a"]
        assert p["smem"] == 4 * (2 * 16 * p["a_ld"] + 2 * 16 * p["BN"]) <= SMEM_ATTR
        assert p["grid"] == (-(-L // p["BM"]), -(-Cout // p["BN"]))
        n += 1
    assert n > 1000


def test_plan_rejects_what_the_launcher_rejects(lib):
    ok = am_plans.conv1d_plan
    assert ok(lib, 2, 300, 48, 64, 3) is not None
    assert ok(lib, 2, 300, 40, 64, 3) is None and b"Cin=40" in lib.ev_last_error()        # C_in % 16
    assert ok(lib, 2, 300, 0, 64, 3) is None
    assert ok(lib, 2, 300, 48, 66, 3) is None and b"Cout=66" in lib.ev_last_error()       # C_out % 4
    assert ok(lib, 2, 300, 48, 64, 4) is None and b"K=4" in lib.ev_last_error()           # even K
    assert ok(lib, 2, 300, 48, 64, 3, 0) is None
    assert ok(lib, 0, 300, 48, 64, 3) is None and ok(lib, 2, 0, 48, 64, 3) is None and ok(lib, 65536, 1, 48, 64, 3) is None
    # the A tile: BM + (K - 1) * dil rows, at most 384 (rows_a is even for odd K: 384 is accepted, 386 the first rejected)
    p = ok(lib, 1, 700, 32, 32, 3, 64)
    assert p is not None and p["BM"] == 256 and p["rows_a"] == 384
    assert ok(lib, 1, 700, 32, 32, 3, 65) is None and b"rows_a=386" in lib.ev_last_error()
    assert ok(lib, 1, 20000, 64, 64, 11, 26) is None and ok(lib, 1, 20000, 64, 64, 11, 25)["rows_a"] == 378


def test_variant_is_a_function_of_batch_length_and_cout(lib):
    shapes = [(16, 1, 1), (64, 3, 1), (384, 3, 1), (1536, 3, 1), (32, 11, 5), (128, 7, 3), (512, 7, 1)]
    for B, L, Cout in itertools.product((1, 2, 3, 8, 32, 64), (1, 63, 64, 65, 128, 129, 1100, 1792, 1793, 2148, 19200),
                                        (32, 48, 64, 80, 128, 384, 1152, 1536, 2048)):
        keys = {am_plans.conv1d_plan(lib, B, L, Cin, Cout, K, dil)["key"] for Cin, K, dil in shapes}
        assert len(keys) == 1, (B, L, Cout, keys)


def test_small_problem_switch(lib):
    """The variants on both sides of each switch at 132 SMs (the examples of the operator cases)."""
    v = lambda *a: am_plans.conv1d_plan(lib, *a)["key"][1:]
    assert v(1, 1100, 384, 1152, 1) == (16, 1, 4) and v(1, 2148, 384, 1152, 1) == (16, 2, 8)
    assert v(1, 1100, 384, 1536, 3) == (16, 1, 4) and v(1, 2148, 384, 1536, 3) == (16, 2, 8)
    assert v(32, 200, 384, 384, 1) == (16, 2, 8) and v(32, 200, 384, 80, 1) == (16, 1, 4)
    assert v(1, 128 * 131, 64, 64, 3) == (16, 1, 4) and v(1, 128 * 132, 64, 64, 3) == (16, 1, 8)
    assert v(1, 128, 64, 64, 3) == (16, 1, 4) and v(64, 19200, 32, 32, 11, 5) == (8, 1, 8)


def test_operator_cases_launch_every_engine_variant_and_pair(lib):
    ck, cp = ffma_cases.case_pairs(lib)
    ek, ep = ffma_cases.engine_pairs(lib)
    assert not ek - ck, "engine (layer, variant) without an operator case: %s" % sorted(ek - ck)
    assert not ep - cp, "engine (layer, batch variant, batch-1 variant) without an operator case: %s" % sorted(ep - cp)
    assert {k[1][1:] for k in ek} == {(8, 1, 8), (16, 1, 4), (16, 1, 8), (16, 2, 8)}
    assert any(pb != p1 for _, pb, p1 in ep)
    # every (k, dil) of c1 and every accumulate mode of c2 at each of the vocoder's widths
    cases = ffma_cases.conv_cases()
    for C in (256, 128, 64, 32):
        assert {(c["K"], c["dil"]) for c in cases if c["layer"] == "c1_C%d" % C} >= set(itertools.product((3, 7, 11), (1, 3, 5)))
        assert {c["acc"] for c in cases if c["layer"] == "c2_C%d" % C} == {0, 1, 2}


def test_case_lists_cover_the_issue_edges():
    cases = {c["name"]: c for c in ffma_cases.conv_cases()}
    assert len(cases) == len(ffma_cases.conv_cases())
    for kind in ("qkv", "wo", "ffn1", "ffn2", "cond.wx", "pred", "to_mel"):
        big = [c for c in cases.values() if c["layer"] == kind and c["B"] == 32]
        assert big and all({1, 63, 64, 65, 127, 128, 129} <= set(ffma_cases.valid_rows(c)) for c in big)
    assert cases["len1_C32_k11_d5"]["units"][-1] == 1 and cases["cin16"]["Cin"] == 16 and cases["cout48"]["Cout"] == 48


@pytest.mark.parametrize("prec", ["fp32_ffma"])
def test_launch_list_rules(lib, prec):
    for B, T, F in ((1, 100, 537), (3, 23, 94), (32, 200, 1100)):
        for inv in (1, 0):
            ls = am_plans.engine_launches(lib, B, T, F, prec, inv)
            assert ("splitk_reduce",) not in ls and ("attention",) in ls and not any(k[0] == "attention_tc" for k in ls)
            convs = [r for r in am_plans.am_layers(B, T, F, prec, inv) if isinstance(r, dict)]
            assert {r["mode"] for r in convs} == {am_plans.FFMA}
            assert sum(k[0] == "conv1d_tm" for k in ls) == len(convs)
    cf = voc_plans.engine_launches(lib, 2, 300, am_plans.FFMA)
    tm = voc_plans.engine_launches(lib, 2, 300, am_plans.FFMA, time_major=True)
    assert cf[0] == ("transpose",) and cf[1:] == tm and tm[-1] == ("conv_post",)
    assert len(tm) == 2 + 4 + 4 * 9 * 2
