"""Host-only checks of the acoustic model's kernel tests themselves (no GPU):

* every tile plan ev_am_phase1 / ev_am_phase2 launch for the reference configuration -- (layer, MODE, MT, KBG, BN, rings,
  producer groups, K-split) at the benchmark's acoustic workloads, in every precision and for literal and batch-invariant
  batches -- is the plan of at least one operator case of tests/test_am_kernels_gpu.py;
* the per-element bound of tests/am_ref.py rejects what it must: a K-split slice dropped for one tile or counted twice, the
  previous item's bias row, a tap missing next to an item end, a key at klen - 1 dropped from the softmax or the key at klen let
  in, tf32-rounded operands judged as fp32-accurate, a NaN in a valid row; and accepts the tf32-rounded results as 1xTF32, the
  lazily rescaled softmax included -- which it would reject without the score term of the attention magnitude;
* the item lengths of the operator cases land where they are meant to: on the 128-row tile edges.
"""
import math

import pytest
import torch

import am_cases
import am_plans
import am_ref
from emotivoice_b200 import packing

PRECS = ("fp32", "tf32", "bf16")
# (workload, B, T phonemes, F frames): the headline (B = 1, 100 phonemes), the fixtures (b1_t12 / t50 / t100, b3_padded), a
# B = 32 batch of 20-200 phonemes and cfg5's B = 32 length buckets, at the frame counts their durations give (~5.4 per phoneme;
# a spread around it for the batches)
WORKLOADS = ([("headline", 1, 100, 537), ("b1_t12", 1, 12, 58), ("b1_t50", 1, 50, 249), ("b1_t100", 1, 100, 537),
              ("b3_padded", 3, 23, 94)]
             + [("b32_mixed", 32, 200, F) for F in (700, 900, 1100, 1300)]
             + [("cfg5_bucket", 32, T, F) for T in (40, 80, 120, 160, 200) for F in (int(4.5 * T), int(6.5 * T))])


def _engine_keys(lib):
    keys = {}
    for name, B, T, F in WORKLOADS:
        for prec in PRECS:
            for inv in (1, 0):
                for k in am_plans.engine_conv_keys(lib, B, T, F, prec, inv):
                    keys.setdefault(k, "%s (B=%d T=%d F=%d, %s)" % (name, B, T, F, prec))
    return keys


def test_every_engine_tile_plan_is_an_operator_case(lib):
    eng = _engine_keys(lib)
    cases = am_cases.case_plans(lib)
    missing = {k: v for k, v in eng.items() if k not in cases}
    assert not missing, "engine plans without an operator case (and a workload that issues them): %s" % missing
    plans = [k for _, k in eng]
    # every K-split factor, kernel MODE and N tile width the acoustic model launches
    assert {p[7] for p in plans} == {2, 4, 8, 16}
    assert {p[0] for p in plans} == {0, 1, 2, 3}
    assert {p[3] for p in plans} == {32, 64, 80, 128}
    assert {p[1] for p in plans} == {1}


def test_launch_list_rules():
    """The literal batch adds mask_rows; the prefix is 3xTF32 in every precision, the decoder and to_mel run the precision's
    MODE."""
    lay = {prec: am_plans.am_layers(1, 100, 537, prec, 1) for prec in PRECS}
    for prec, ls in lay.items():
        convs = [r for r in ls if isinstance(r, dict)]
        assert all(r["mode"] == 1 for r in convs if not r["name"].startswith(("dec.", "to_mel")))
        assert {r["mode"] for r in convs if r["name"].startswith(("dec.", "to_mel"))} == {am_plans.decoder_mode(prec)}
    lit = am_plans.am_layers(3, 23, 94, "fp32", 0)
    assert ("mask_rows",) in lit and ("mask_rows",) not in am_plans.am_layers(3, 23, 94, "fp32", 1)


def test_uneven_slices_are_planned(lib):
    """bf16x3 / bf16 wo and ffn1 of the decoder: 6 C_in blocks of 64 channels over S = 4 (slices of 1, 2, 1, 2 blocks)."""
    for mode in (2, 3):
        p = am_plans.tc_plan(lib, 1, 537, 384, 384, 1, mode, 4)
        assert p["KBG"] == 8 and p["S"] == 4


# ---- the checker rejects the faults it must catch ------------------------------------------------------------------------
def _conv_case(seed=3, B=2, L=300, Cin=64, Cout=48, K=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, Cin, generator=g)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    bias = torch.randn(B, Cout, generator=g)
    return x, w, bias


@pytest.mark.parametrize("mode", (0, 1, 2, 3))
def test_bound_rejects_a_k_split_slice_dropped_or_counted_twice(mode):
    x, w, bias = _conv_case()
    n, S, KB = 300, 4, 16          # C_in blocks of 16 channels, slice z = blocks [z n_cb / S, (z + 1) n_cb / S)
    y64, m = am_ref.conv_ref(x[0], w, bias[0], None, n)
    assert am_ref.check(y64, y64, m, mode)["ok"]
    n_cb = w.shape[1] // KB
    z = 2
    c0, c1 = z * n_cb // S * KB, (z + 1) * n_cb // S * KB
    ws = torch.zeros_like(w)
    ws[:, c0:c1] = w[:, c0:c1]
    part, _ = am_ref.conv_ref(x[0], ws, None, None, n)
    t0, t1, n0, n1 = 128, 256, 0, 32         # one output tile
    for sign in (-1, 1):
        bad = y64.clone()
        bad[t0:t1, n0:n1] += sign * part[t0:t1, n0:n1]
        r = am_ref.check(bad, y64, m, mode)
        assert not r["ok"] and r["err_m"] > am_ref.TAU[mode], (sign, r)


@pytest.mark.parametrize("mode", (0, 1, 2, 3))
def test_bound_rejects_the_previous_items_bias_row(mode):
    x, w, bias = _conv_case()
    y64, m = am_ref.conv_ref(x[1], w, bias[1], None, 200)
    bad, _ = am_ref.conv_ref(x[1], w, bias[0], None, 200)
    assert not am_ref.check(bad, y64, m, mode)["ok"]


@pytest.mark.parametrize("act", (am_ref.ACT_NONE, am_ref.ACT_RELU, am_ref.ACT_GELU))
@pytest.mark.parametrize("mode", (0, 1, 2, 3))
def test_bound_rejects_a_missing_tap_next_to_an_item_end(mode, act):
    x, w, bias = _conv_case(K=3)
    n = 129
    x[0, n:] = float("nan")
    y64, m = am_ref.conv_ref(x[0], w, bias[0], None, n, act)
    # row n - 1: tap 2 reads row n (padding); drop tap 0 (row n - 2), which reads a valid row
    wd = w.clone()
    wd[0] = 0
    alt, _ = am_ref.conv_ref(x[0], wd, bias[0], None, n, act)
    bad = y64.clone()
    bad[n - 1] = alt[n - 1]
    r = am_ref.check(bad, y64, m, mode)
    assert not r["ok"] and r["err_m"] > am_ref.TAU[mode], r


def test_bound_rejects_tf32_operands_as_fp32_accurate_and_accepts_them_as_tf32():
    g = torch.Generator().manual_seed(5)
    n, Cin, Cout, K = 200, 1536, 64, 3      # the ffn2 reduction: 4608 terms
    x = torch.randn(n, Cin, generator=g)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g)
    res = torch.randn(n, Cout, generator=g)
    for act in (am_ref.ACT_NONE, am_ref.ACT_GELU):
        y64, m = am_ref.conv_ref(x, w, b, res, n, act)
        y_tf, _ = am_ref.conv_ref(packing.round_tf32(x), packing.round_tf32(w), b, res, n, act)
        for mode in (1, 3):
            assert not am_ref.check(y_tf, y64, m, mode)["ok"]
        assert am_ref.check(y_tf, y64, m, 0)["ok"]


def test_bound_rejects_a_nan_in_a_valid_row():
    x, w, bias = _conv_case()
    y64, m = am_ref.conv_ref(x[0], w, bias[0], None, 300)
    bad = y64.clone()
    bad[299, 5] = float("nan")
    for mode in (0, 1, 2, 3):
        assert not am_ref.check(bad, y64, m, mode)["ok"]
    o64, om = am_ref.attn_ref(torch.randn(50, 3 * 384), 50, 8)
    bad = o64.clone()
    bad[49, 0] = float("nan")
    assert not am_ref.check(bad, o64, om, 0, am_ref.ATTN_REL_MAX[0])["ok"]


def _qkv(L, seed=11):
    return torch.randn(L, 3 * 384, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("mode", (0, 1))
def test_bound_rejects_a_key_dropped_or_let_in_at_klen(mode):
    L, klen = 200, 129
    qkv = _qkv(L)
    o64, m = am_ref.attn_ref(qkv, klen, 8)
    assert am_ref.check(o64, o64, m, mode, am_ref.ATTN_REL_MAX[mode])["ok"]
    dropped, _ = am_ref.attn_ref(qkv, klen - 1, 8, rows=torch.arange(klen))         # the key at klen - 1 left out
    let_in, _ = am_ref.attn_ref(qkv, klen + 1, 8, rows=torch.arange(klen))          # the key at klen taken in
    for bad in (dropped, let_in):
        r = am_ref.check(bad, o64, m, mode, am_ref.ATTN_REL_MAX[mode])
        assert not r["ok"] and r["err_m"] > am_ref.TAU[mode], r


def _lazy_qkv(L=400):
    """test_attention_tc_lazy_rescale_path's construction: keys of later 64-key tiles grow past the rescale threshold."""
    qkv = _qkv(L, seed=77)
    qkv[:, 384:768] *= (1.0 + 2.5 * (torch.arange(L) // 64).float())[:, None]
    qkv[1::3, :384] *= 0.05
    return qkv


def _tf32_attention(qkv, klen):
    """The attention on tf32-rounded q, k, v (in fp64 otherwise): the operand error of one tf32 MMA per K step."""
    t = qkv.clone()
    t[:klen] = packing.round_tf32(t[:klen])
    return am_ref.attn_ref(t, klen, 8, score_term=False)[0]


@pytest.mark.parametrize("lazy", (False, True))
def test_attention_bound_rejects_tf32_operands_as_fp32_accurate_and_accepts_them_as_tf32(lazy):
    L, klen = 400, 333
    qkv = _lazy_qkv(L) if lazy else _qkv(L)
    o64, m = am_ref.attn_ref(qkv, klen, 8)
    y = _tf32_attention(qkv, klen)
    rel0 = (am_ref.ATTN_REL_MAX_LARGE_SCORES if lazy else am_ref.ATTN_REL_MAX)[0]
    assert am_ref.check(y, o64, m, 0, rel0)["ok"]
    assert not am_ref.check(y, o64, m, 1, am_ref.ATTN_REL_MAX[1])["ok"]


def test_attention_bound_needs_the_score_term():
    """Without the softmax term of m the tf32 result of the lazily rescaled case (scores of ~100) is out of the 1xTF32 bound."""
    L, klen = 400, 333
    qkv = _lazy_qkv(L)
    o64, m_no = am_ref.attn_ref(qkv, klen, 8, score_term=False)
    y = _tf32_attention(qkv, klen)
    assert not am_ref.check(y, o64, m_no, 0, am_ref.ATTN_REL_MAX_LARGE_SCORES[0])["ok"]


def test_operator_case_lengths_land_on_tile_edges():
    for L in (am_cases.PREFIX_L32, am_cases.DEC_L32):
        lens = am_cases.ragged_lens(L)
        assert len(lens) == am_cases.B32 and max(lens) == L and min(lens) == 1
        assert {n % 128 for n in lens} >= {0, 1, 127} and {63, 64, 65} <= set(lens)
    att = [c for c in am_cases._attn_cases() if c["B"] == am_cases.B32][0]
    assert {1, 63, 64, 65, 127, 128, 129, att["L"]} <= set(att["lens"]) and len(att["lens"]) == am_cases.B32
    # batch-1 decoder lengths: one, two, five and nine 128-row tiles, each ragged in its last tile
    assert [-(-L // 128) for L in am_cases.DEC_L1["wo"]] == [1, 5, 9]
