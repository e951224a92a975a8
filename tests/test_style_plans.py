"""Host-only checks of the style encoder's GEMM tests themselves (no GPU):

* every tile plan ev_style_forward launches -- (layer, MODE, MT, KBG, BN, rings, producer groups, K-split) for BERT-base and the
  small model, in "fp32" and "tf32", at every token count up to max_position and batches of 1 to 128 -- is the plan of at
  least one operator case of tests/test_style_kernels_gpu.py (the style family of tests/am_cases.py);
* the launch list of tests/style_plans.py follows the rules of style_engine.cu;
* the per-element bound of tests/am_ref.py rejects, at the style shapes, the faults a split-K GEMM can make, emulated in fp32: a
  K slice dropped or counted twice in one output tile, the GELU or the residual applied per slice, one slice of a 3xTF32 ffn2
  without its lo plane, the last of qkv's 18 N tiles reading the 17th tile's weights -- and accepts the faultless emulation;
* the operator cases' item lengths land on the 128-row edges and on every N tile width change.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import am_cases
import am_plans
import am_ref
import style_plans
from emotivoice_b200 import packing

PRECS = ("fp32", "tf32")
BATCHES = (1, 2, 3, 4, 8, 16, 32, 64, 128)


def _max_tokens(cfg):
    return int(style_plans.style_config(cfg).max_position_embeddings)


def _engine_keys(lib, cfg):
    keys = {}
    for prec in PRECS:
        for B in BATCHES:
            for N in range(1, _max_tokens(cfg) + 1):
                for k in style_plans.style_conv_keys(lib, cfg, B, N, prec):
                    keys.setdefault(k, "B=%d N=%d %s" % (B, N, prec))
    return keys


@pytest.mark.parametrize("cfg", style_plans.CONFIGS)
def test_every_style_tile_plan_is_an_operator_case(lib, cfg):
    eng = _engine_keys(lib, cfg)
    cases = am_cases.case_plans(lib, "style")
    missing = {k: v for k, v in eng.items() if k not in cases}
    assert not missing, "style plans without an operator case (and a call that issues them): %s" % missing
    plans = {k for _, k in eng}
    assert {p[0] for p in plans} == {0, 1} and {p[7] for p in plans} == {2, 4} and {p[3] for p in plans} == {32, 64, 128}
    # the plans the acoustic model's cases never launch: 3xTF32 at S = 2 (the fp32 style encoder's qkv, wo and ffn1)
    am_keys = {k for _, k in am_cases.case_plans(lib, "tc")}
    new = {p for p in plans - am_keys if p[0] == 1 and p[7] == 2}
    assert {p[3] for p in new} == {32, 64, 128}, sorted(plans - am_keys)


def test_launch_list_rules(lib):
    for cfg in style_plans.CONFIGS:
        n_layers = int(style_plans.style_config(cfg).num_hidden_layers)
        for prec in PRECS:
            ls = style_plans.style_layers(cfg, 3, 100, prec)
            convs = [r for r in ls if isinstance(r, dict)]
            assert len(convs) == 4 * n_layers
            assert {r["mode"] for r in convs} == {style_plans.style_mode(prec)}
            assert {r["kind"].split(".")[-1]: r["ksplit"] for r in convs} == {"qkv": 2, "wo": 2, "ffn1": 2, "ffn2": 4}
            assert {r["kind"].split(".")[-1] for r in convs if r["out_act"] == am_plans.ACT_GELU} == {"ffn1"}
            assert {r["kind"].split(".")[-1] for r in convs if r["res"]} == {"wo", "ffn2"}
            for B, N in ((1, 1), (1, 20), (3, 129), (32, 512)):
                N = min(N, _max_tokens(cfg))
                full = style_plans.style_launches(lib, cfg, B, N, prec)
                bare = style_plans.style_launches(lib, cfg, B, N, prec, heads=False)
                # every GEMM is followed by its reduce: the clamped S stays > 1 at every style shape
                idx = [i for i, r in enumerate(full) if r[0] in (0, 1)]
                assert len(idx) == 4 * n_layers and all(full[i + 1] == ("splitk_reduce",) for i in idx)
                assert all(full[i][7] == (4 if j % 4 == 3 else 2) for j, i in enumerate(idx))
                assert full[:2] == [("validate_inputs",), ("bert_embed_ln",)]
                assert full[-2:] == [("row_gemv", "pooler"), ("row_gemv", "heads")] and bare == full[:-1]
                assert len(full) == 2 + 11 * n_layers + 2
    assert len(style_plans.style_launches(lib, "base", 1, 20, "fp32")) == 136
    assert len(style_plans.style_launches(lib, "small", 1, 20, "fp32")) == 26


# ---- the checker rejects the faults a split-K style GEMM can make --------------------------------------------------------
N_ROWS = 130          # two 128-row tiles, the second ragged


def _gemm_case(cfg, kind, seed=3, n=N_ROWS):
    """Inputs of one style GEMM at its real C_in / C_out (am_cases' magnitudes): x (n, Cin), w (Cin, Cout), bias, residual."""
    Cin, Cout, _, act, res_kind, _, gelu_in = am_cases.LAYERS[style_plans.kind_name(cfg, kind)]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, Cin, generator=g)
    x = F.gelu(x) if gelu_in else x
    w = torch.randn(Cin, Cout, generator=g) / math.sqrt(Cin)
    bias = torch.randn(Cout, generator=g)
    res = torch.randn(n, Cout, generator=g) if res_kind else None
    return x, w, bias, res, act


def _slices(lib, cfg, kind, mode):
    """Channel ranges [c0, c1) of the K slices: blocks [z n_cb / S, (z + 1) n_cb / S) of KB = 4 * KBG channels (conv1d_tc)."""
    Cin, Cout = am_cases.LAYERS[style_plans.kind_name(cfg, kind)][:2]
    p = am_plans.tc_plan(lib, 1, N_ROWS, Cin, Cout, 1, mode, style_plans.SPLITS[kind])
    KB = 4 * p["KBG"]
    n_cb, S = Cin // KB, p["S"]
    return [(z * n_cb // S * KB, (z + 1) * n_cb // S * KB) for z in range(S)]


def _partials(x, w, mode, slices, no_lo=()):
    """fp32 partial sums of the K slices as the MODE forms its products: 1xTF32 = tf32 operands; 3xTF32 = hi hi + hi lo + lo hi
    (hi = tf32(v), lo = tf32(v - hi)), except in the slices of `no_lo`, which keep hi hi alone."""
    xh, wh = packing.round_tf32(x), packing.round_tf32(w)
    xl, wl = packing.round_tf32(x - xh), packing.round_tf32(w - wh)
    out = []
    for z, (c0, c1) in enumerate(slices):
        p = xh[:, c0:c1] @ wh[c0:c1]
        if mode == 1 and z not in no_lo:
            p = p + (xh[:, c0:c1] @ wl[c0:c1] + xl[:, c0:c1] @ wh[c0:c1])
        out.append(p)
    return out


def _act(y, act):
    return F.gelu(y) if act == am_plans.ACT_GELU else y


def _reduce(parts, bias, act, res):
    """splitk_reduce_store: the slices in the order z = 0..S-1, then bias, activation, residual."""
    y = torch.zeros_like(parts[0])
    for p in parts:
        y = y + p
    y = _act(y + bias, act)
    return y if res is None else y + res


def _ref(x, w, bias, res, act):
    return am_ref.conv_ref(x, w[None], bias, res, x.shape[0], act)


def _rejects(bad, y64, m, mode):
    r = am_ref.check(bad, y64, m, mode)
    return not r["ok"], r


@pytest.mark.parametrize("mode", (1, 0))
@pytest.mark.parametrize("kind", style_plans.KINDS)
def test_bound_accepts_the_faultless_split_k_emulation(lib, kind, mode):
    x, w, bias, res, act = _gemm_case("base", kind)
    y64, m = _ref(x, w, bias, res, act)
    y = _reduce(_partials(x, w, mode, _slices(lib, "base", kind, mode)), bias, act, res)
    r = am_ref.check(y, y64, m, mode)
    assert r["ok"], r


@pytest.mark.parametrize("mode", (1, 0))
@pytest.mark.parametrize("kind", ("qkv", "wo", "ffn1"))
def test_bound_rejects_an_s2_slice_dropped_or_counted_twice(lib, kind, mode):
    """One CTA's slice of one 128 x 128 output tile (the second, ragged row tile) lost, or added twice."""
    x, w, bias, res, act = _gemm_case("base", kind)
    y64, m = _ref(x, w, bias, res, act)
    sl = _slices(lib, "base", kind, mode)
    assert len(sl) == 2
    for z in range(2):
        for scale in (0.0, 2.0):
            parts = _partials(x, w, mode, sl)
            parts[z][128:, 0:128] *= scale
            bad, r = _rejects(_reduce(parts, bias, act, res), y64, m, mode)
            assert bad and r["err_m"] > am_ref.TAU[mode], (z, scale, r)


@pytest.mark.parametrize("mode", (1, 0))
def test_bound_rejects_the_gelu_applied_per_slice(lib, mode):
    """ffn1's epilogue (bias, GELU) run on each slice's partial sum, the reduce only adding them."""
    x, w, bias, res, act = _gemm_case("base", "ffn1")
    y64, m = _ref(x, w, bias, res, act)
    parts = _partials(x, w, mode, _slices(lib, "base", "ffn1", mode))
    bad = sum(_act(p + bias, act) for p in parts)
    rej, r = _rejects(bad, y64, m, mode)
    assert rej and r["err_m"] > am_ref.TAU[mode], r


@pytest.mark.parametrize("mode", (1, 0))
@pytest.mark.parametrize("kind", ("wo", "ffn2"))
def test_bound_rejects_the_residual_added_once_per_slice(lib, kind, mode):
    x, w, bias, res, act = _gemm_case("base", kind)
    y64, m = _ref(x, w, bias, res, act)
    parts = _partials(x, w, mode, _slices(lib, "base", kind, mode))
    bad = _reduce(parts, bias, act, res) + (len(parts) - 1) * res
    rej, r = _rejects(bad, y64, m, mode)
    assert rej and r["err_m"] > am_ref.TAU[mode], r


@pytest.mark.parametrize("z", (0, 3))
def test_bound_rejects_one_ffn2_slice_without_its_lo_plane(lib, z):
    """A 3xTF32 ffn2 (C_in 3072, S = 4) with one K slice computed from tf32 operands: a 1xTF32-sized error on a quarter of the
    reduction.  Random rounding errors stay below the worst-case tau * m (err/m ~2^-15 here), so it is the bound relative to
    max|y64| that rejects it, on a full 512-token item -- as it rejects tf32 operands in the whole reduction; the 1xTF32 bound
    accepts it."""
    x, w, bias, res, act = _gemm_case("base", "ffn2", n=512)
    y64, m = _ref(x, w, bias, res, act)
    sl = _slices(lib, "base", "ffn2", 1)
    assert len(sl) == 4 and sl[-1][1] == 3072
    bad = _reduce(_partials(x, w, 1, sl, no_lo=(z,)), bias, act, res)
    rej, r = _rejects(bad, y64, m, 1)
    assert rej, r
    assert am_ref.check(bad, y64, m, 0)["ok"]


@pytest.mark.parametrize("mode", (1, 0))
def test_bound_rejects_the_last_qkv_tile_reading_the_previous_tiles_weights(lib, mode):
    x, w, bias, res, act = _gemm_case("base", "qkv")
    assert w.shape[1] == 18 * 128
    y64, m = _ref(x, w, bias, res, act)
    wb = w.clone()
    wb[:, 17 * 128:] = w[:, 16 * 128:17 * 128]
    bad = y64.clone()
    bad[:, 17 * 128:] = _reduce(_partials(x, wb, mode, _slices(lib, "base", "qkv", mode)), bias, act, res)[:, 17 * 128:]
    rej, r = _rejects(bad, y64, m, mode)
    assert rej and r["err_m"] > am_ref.TAU[mode], r


# ---- the case lengths ----------------------------------------------------------------------------------------------------
def test_style_case_lengths_land_on_tile_edges_and_bn_thresholds(lib):
    cases = am_cases._style_cases()
    for cfg in style_plans.CONFIGS:
        L1 = am_cases.STYLE_L1[cfg]
        nmax = _max_tokens(cfg)
        assert max(L1) == nmax and min(L1) == 1 and {n % 128 for n in L1} >= {0, 1}
        for kind in style_plans.KINDS:
            Cin, Cout = am_cases.LAYERS[style_plans.kind_name(cfg, kind)][:2]
            for mode in (1, 0):
                bn = {N: am_plans.tc_plan(lib, 1, N, Cin, Cout, 1, mode, style_plans.SPLITS[kind])["BN"] for N in range(1, nmax + 1)}
                # both sides of every change of the batch-1 N tile width are case lengths
                for N in range(2, nmax + 1):
                    if bn[N] != bn[N - 1]:
                        assert N - 1 in L1 and N in L1, (cfg, kind, mode, N)
                assert {bn[N] for N in L1} == set(bn.values())
        for B, head in am_cases.STYLE_RAGGED[cfg]:
            cs = [c for c in cases if c["kind"].startswith(cfg + ":") and c["B"] == B]
            assert len(cs) == 8
            for c in cs:
                assert len(c["lens"]) == B and max(c["lens"]) == c["L"] == head[0] and min(c["lens"]) >= 1
                assert c["lens"][:len(head)] == list(head) and c["edges"] == len(head)
    base = dict(am_cases.STYLE_RAGGED["base"])
    assert {64, 1, 2, 31, 32, 33, 63} <= set(base[32]) and {512, 1, 127, 128, 129, 255, 256, 257} <= set(base[8])
    assert {n % 128 for n in base[8]} >= {0, 1, 127}
    # the ragged batches run at BN = 128 (base); the small model's at 128, 64 and 32 as well
    for cfg, want in (("base", {128}), ("small", {32, 64, 128})):
        got = set()
        for c in cases:
            if c["kind"].startswith(cfg + ":") and c["B"] > 1:
                Cin, Cout = am_cases.LAYERS[c["kind"]][:2]
                got.add(am_plans.tc_plan(lib, c["B"], c["L"], Cin, Cout, 1, c["mode"], c["S"])["BN"])
        assert got == want, (cfg, got)
