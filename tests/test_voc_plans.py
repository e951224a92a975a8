"""Host-only checks of the vocoder kernel tests themselves (no GPU):

* every tile plan ev_vocoder can launch for the reference configuration -- (kernel, MODE, MT, KBG, BN, rate) over batch sizes
  and lengths spanning its regimes -- is the plan of at least one operator case of tests/test_voc_kernels_gpu.py, so no
  template instantiation the engine runs goes unchecked against fp64;
* the per-element bound of tests/voc_ref.py rejects what it must: a missing tap at an item end, a result with tf32-rounded
  operands judged as fp32-accurate, a NaN in a valid row; and accepts what it must (the tf32-rounded result in mode 0);
* the item lengths of the operator cases land where they are meant to: on tile edges.
"""
import math

import pytest
import torch

import voc_cases
import voc_plans
import voc_ref
from emotivoice_b200 import packing

GRID_B = (1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64)
GRID_F = (1, 8, 20, 40, 60, 100, 150, 200, 300, 400, 540, 700, 900, 1024, 1100, 1500, 2000, 3000, 4096)


def _engine_keys(lib):
    sh = voc_plans.voc_shapes()
    keys = {}
    for B in GRID_B:
        for F in GRID_F:
            for mode in voc_cases.MODES:
                for k in voc_plans.engine_launches(lib, B, F, mode, sh):
                    if len(k) > 1:
                        keys.setdefault(k, (B, F))
    return keys


def test_every_engine_tile_plan_is_an_operator_case(lib):
    eng = _engine_keys(lib)
    cases = set()
    for fam in ("conv", "pair", "group", "pair_group"):
        cases |= voc_cases.case_plans(lib, fam)
    missing = {k: v for k, v in eng.items() if k not in cases}
    assert not missing, "engine plans without an operator case (first (B, F) that issues them): %s" % missing
    # all four kernels, every mode, one to four accumulators per tile
    assert {k[0] for k in eng} == {"conv1d_gp", "conv1d_gp_group", "resblock_gp", "resblock_gp_group"}
    assert {k[1] for k in eng} == {0, 1, 2, 3} and {k[2] for k in eng} == {1, 2, 4}


def test_the_launch_list_spans_the_vocoders_regimes(lib):
    """Grouped launches + the sum pass at small B*F; above 2400 batch-frames one launch per layer, fused where the fused plan
    keeps two accumulators per tile, and the 64-channel k11 layers (B * L > 280 000) as two launches."""
    sh = voc_plans.voc_shapes()
    small = voc_plans.engine_launches(lib, 1, 1024, 3, sh)
    assert ("gp_sum_div",) in small and any(k[0] == "conv1d_gp_group" for k in small)
    mid = voc_plans.engine_launches(lib, 4, 1050, 3, sh)
    assert not any(k[0].endswith("_group") for k in mid) and any(k[0] == "resblock_gp" for k in mid)
    big = voc_plans.engine_launches(lib, 8, 700, 3, sh)
    n_conv = lambda ks: sum(k[0] == "conv1d_gp" for k in ks)
    assert n_conv(big) >= n_conv(mid) > 0


def _case(seed=3, n=300, L=400, Cin=32, Cout=32, K=7, dil=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(L, Cin, generator=g)
    x[n:] = float("nan")
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    bias = torch.randn(Cout, generator=g)
    return x, w, bias


@pytest.mark.parametrize("mode", voc_cases.MODES)
def test_bound_rejects_a_missing_tap_next_to_an_item_end(mode):
    n, K, dil = 300, 7, 3
    x, w, bias = _case(n=n, K=K, dil=dil)
    y64, m = voc_ref.conv_ref(x, w, bias, None, None, n, 0, n, dil)
    assert voc_ref.check(y64, y64, m, mode)["ok"]
    # row n-2: taps j with r + (j-3)*dil >= n read the zero padding; drop tap 2 (row n-5), which reads a valid row
    r, j = n - 2, 2
    xa = voc_ref.lrelu(x[:n].double())
    contrib = xa[r + (j - (K - 1) // 2) * dil] @ w[j].double()
    bad = y64.clone()
    bad[r] -= contrib
    res = voc_ref.check(bad, y64, m, mode)
    assert not res["ok"] and res["err_m"] > voc_ref.TAU[mode], res


def test_bound_rejects_tf32_operands_as_fp32_accurate_and_accepts_them_as_tf32():
    n, K, dil = 300, 11, 1
    x, w, bias = _case(seed=5, n=n, K=K, dil=dil, Cin=64, Cout=64)
    y64, m = voc_ref.conv_ref(x, w, bias, None, None, n, 0, n, dil)
    xr = packing.round_tf32(voc_ref.lrelu(x[:n]).float())
    y_tf, _ = voc_ref.conv_ref(xr, packing.round_tf32(w), bias, None, None, n, 0, n, dil, act=False)
    for mode in (1, 3):
        assert not voc_ref.check(y_tf, y64, m, mode)["ok"]
    assert voc_ref.check(y_tf, y64, m, 0)["ok"]


def test_bound_rejects_a_nan_in_a_valid_row():
    x, w, bias = _case()
    y64, m = voc_ref.conv_ref(x, w, bias, None, None, 300, 0, 300, 3)
    bad = y64.clone()
    bad[299, 5] = float("nan")
    for mode in voc_cases.MODES:
        assert not voc_ref.check(bad, y64, m, mode)["ok"]


def test_fused_reference_is_two_convolutions_and_windows_match_whole_items():
    n, K, dil, C = 200, 7, 5, 32
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, C, generator=g)
    w1 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
    w2 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
    b1, b2 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xt, _ = voc_ref.conv_ref(x, w1, b1, None, None, n, 0, n, dil)
    y, _ = voc_ref.conv_ref(xt, w2, b2, x, None, n, 0, n, 1)
    yp, mp = voc_ref.pair_ref(x, w1, b1, w2, b2, None, n, 0, n, dil)
    assert torch.allclose(y, yp, rtol=0, atol=1e-12) and bool((mp >= yp.abs()).all())
    for r0, r1 in voc_ref.windows(n, 64, width=20, edge=30):
        yw, _ = voc_ref.pair_ref(x, w1, b1, w2, b2, None, n, r0, r1, dil)
        assert torch.allclose(yw, yp[r0:r1], rtol=0, atol=1e-12)


def test_operator_case_lengths_land_on_tile_edges():
    for tile in (128, 256, 512):
        mul = voc_cases.odd_mul(tile)
        lens = voc_cases.pick_lens(7, 40000, tile, voc_cases.CONV_RESIDUES, mul)
        got = [v * mul % tile for v in lens[1:]]
        assert got == list(voc_cases.CONV_RESIDUES), (tile, got)
    R = 512 - 10
    mul = voc_cases.odd_mul(R)
    lens = voc_cases.pick_lens(5, 20000, R, (0, 1, R - 1), mul, tiny=True)
    assert [v * mul % R for v in lens[1:4]] == [0, 1, R - 1] and lens[4] == 1
