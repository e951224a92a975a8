"""Operator cases of the "fp32_ffma" path's kernels, and what ties them to the engine's launches.

* conv1d_tm_kernel<TXN, NV, TM> (conv1d_tm.cu, through ev_op_conv1d): every GEMM-shaped layer of the acoustic model (am_cases.KINDS,
  with the engine's bias, activation and residual) and every convolution of the vocoder (conv_pre, the four polyphase ups, the
  ResBlocks' c1 and c2 with each accumulate mode), at batches whose items fall on both sides of the launcher's variant switches,
  plus the launcher's limits.
* conv_post_kernel (voc_kernels.cu, through ev_op_conv_post).

Every kernel here is one fp32 FFMA chain per output, so every case is held to the fp32-accurate class of tests/voc_ref.py:
|y - y64| <= 2^-14 m per element and 5e-5 of max|y64|.  The longest chain, ffn2's 1536 x 3 = 4608 products, bounds the
accumulation error by 4608 * 2^-24 ~ 2^-11.8 of m in the worst case; rounding errors of random sign grow like its square root
(~2^-20), which is what the bound relies on.

Inputs hold NaN in every row at or past an item's length, residual rows there as well: a kernel that read such a row would turn
a valid output into NaN.  Outputs are prefilled with NaN (with the previous values in the valid rows for ADD / ADD_DIV, with the
residual for an in-place residual); rows past each item must come out as exact zeros.

launch_conv1d picks its variant from (B, L, C_out) and the SM count, so an item inside a batch and the same item alone often run
different variants.  Each case launches every item again at batch 1 and requires the same bits; `case_pairs` lists the
(layer, batch variant, batch-1 variant) pairs the cases exercise and `engine_pairs` those the engine can produce for the
corpus's batches (tests/test_ffma_plans.py holds the first to cover the second).
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(1, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import am_cases  # noqa: E402
import am_plans  # noqa: E402
import voc_plans  # noqa: E402

SLOPE = 0.1
ENGINE_B = (1, 3, 8, 32, 64)
FRAMES_PER_PHONEME = (4.5, 6.5)      # the spread of frame counts the seeded model's durations give (tests/test_am_plans.py)


def _case(name, family, layer, Cin, Cout, K, units, mul=1, dil=1, rate=1, act=0, out_act=0, res=None, acc=0, per_item=False,
          gelu_in=False, lens=True):
    """units: item lengths in units of `mul` rows, passed as lens / lens_mul (lens=False: a null lens pointer, every item L rows)."""
    return dict(name=name, family=family, layer=layer, Cin=Cin, Cout=Cout, K=K, dil=dil, rate=rate, act=act, out_act=out_act, res=res,
                acc=acc, per_item=per_item, gelu_in=gelu_in, units=list(units), mul=mul, lens=lens, B=len(units))


def _am_conv_cases():
    cs = []
    for kind, (Cin, Cout, K, oact, res, per_item, gelu_in) in am_cases.KINDS.items():
        kw = dict(out_act=oact, res=res, per_item=per_item, gelu_in=gelu_in)
        tag = kind.replace(".", "")
        # batch 1 on both sides of the small-problem switch where the engine's lengths reach it (qkv, ffn1 at 2148 frames)
        for L in {"qkv": (1100, 2148), "ffn1": (1100, 2148), "cond.wx": (200,), "pred": (200,)}.get(kind, (1100,)):
            cs.append(_case("%s_B1_L%d" % (tag, L), "am", kind, Cin, Cout, K, [L], lens=False, **kw))
        cs.append(_case("%s_B3_L200" % tag, "am", kind, Cin, Cout, K, [200, 129, 1], **kw))
        cs.append(_case("%s_B32_L200" % tag, "am", kind, Cin, Cout, K, am_cases.ragged_lens(200, seed=len(kind)), **kw))
    Cin, Cout, K = am_cases.KINDS["to_mel"][:3]
    cs.append(_case("tomel_B32_L600", "am", "to_mel", Cin, Cout, K, am_cases.ragged_lens(600, seed=11)))
    return cs


# (C, lens_mul, frames per item) of the ResBlock grid: every (k, dil) of c1 and each accumulate mode of c2, at short items
GRID = ((256, 8, (40, 17, 1)), (128, 64, (12, 5, 1)), (64, 128, (10, 3, 1)), (32, 256, (6, 2, 1)))
# batches whose items take another variant alone than inside the batch: (C, lens_mul, frames, c1 (K, dil), c2 (K, acc))
VARIANT_BATCHES = ((256, 8, (1100, 700, 65, 1), (11, 5), (11, 2)), (128, 64, (300, 262, 70, 1), (11, 5), (7, 1)),
                   (64, 128, (150, 131, 40, 1), (7, 3), (3, 0)))


def _voc_conv_cases():
    sh = voc_plans.voc_shapes()
    cs = [_case("pre_B3_F300", "voc", "pre", sh["n_mels"], sh["c0"], sh["pre_k"], (300, 129, 1)),
          _case("pre_B8_F700", "voc", "pre", sh["n_mels"], sh["c0"], sh["pre_k"], (700, 1, 150, 37, 260, 9, 64, 129))]
    ups_frames = ((1100, 1024, 1), (300, 256, 1), (300, 262, 1), (150, 131, 1))
    mul = 1
    for s, u in enumerate(sh["ups"]):
        cs.append(_case("ups%d_B3_F%d" % (s, ups_frames[s][0]), "voc", "ups%d" % s, u["cin"], u["rate"] * u["cout"], u["K"], ups_frames[s],
                        mul=mul, rate=u["rate"], act=1))
        mul *= u["rate"]
    cs.append(_case("ups3_B1_F1", "voc", "ups3", 64, 64, 3, (1,), mul=128, rate=2, act=1))
    cs.append(_case("ups3_B1_F150", "voc", "ups3", 64, 64, 3, (150,), mul=128, rate=2, act=1))
    for C, m, fr in GRID:
        for K in (3, 7, 11):
            for d in (1, 3, 5):
                cs.append(_case("c1_C%d_k%d_d%d" % (C, K, d), "voc", "c1_C%d" % C, C, C, K, fr, mul=m, dil=d, act=1))
        for K, acc in ((3, 0), (7, 1), (11, 2)):
            cs.append(_case("c2_C%d_k%d_acc%d" % (C, K, acc), "voc", "c2_C%d" % C, C, C, K, fr, mul=m, act=1, res="separate", acc=acc))
    for C, m, fr, (K1, d1), (K2, acc) in VARIANT_BATCHES:
        cs.append(_case("c1_C%d_k%d_d%d_F%d" % (C, K1, d1, fr[0]), "voc", "c1_C%d" % C, C, C, K1, fr, mul=m, dil=d1, act=1))
        cs.append(_case("c2_C%d_k%d_acc%d_F%d" % (C, K2, acc, fr[0]), "voc", "c2_C%d" % C, C, C, K2, fr, mul=m, act=1, res="separate",
                        acc=acc))
    cs.append(_case("c1_C64_k11_d5_B1_F1", "voc", "c1_C64", 64, 64, 11, (1,), mul=128, dil=5, act=1))
    cs.append(_case("c1_C64_k11_d5_B1_F150", "voc", "c1_C64", 64, 64, 11, (150,), mul=128, dil=5, act=1))
    return cs


def _limit_cases():
    """The launcher's limits: a single C_in chunk, a partial 64-wide N tile, the widest accepted A tile (BM 256 + 2 * 64 rows = 384)
    and an item of one row under the widest halo of the vocoder (C 32, k 11, dil 5)."""
    return [_case("cin16", "limit", "cin16", 16, 64, 3, (300, 65)),
            _case("cout48", "limit", "cout48", 64, 48, 5, (300, 129), act=1),
            _case("rows_a_384", "limit", "rows_a_384", 32, 32, 3, (700, 257), dil=64, act=1),
            _case("len1_C32_k11_d5", "limit", "len1", 32, 32, 11, (300, 1), dil=5, act=1, res="separate", acc=2)]


def conv_cases():
    return _am_conv_cases() + _voc_conv_cases() + _limit_cases()


# conv_post: voc_cases._post_cases' shapes (C 32, k 7 and k 5, lens x 256 and none; L not a multiple of 256) and the launcher's
# limits, C = 128 and K = 15 (147,000 of the 160 KB shared-memory attribute)
POST_CASES = [dict(name="k7_B3", B=3, L=5003, C=32, K=7, lens=(20, 13, 1), mul=256),
              dict(name="k7_nolens", B=1, L=1001, C=32, K=7, lens=None, mul=1),
              dict(name="k5_B2", B=2, L=3001, C=32, K=5, lens=(11, 3), mul=256),
              dict(name="C128_k15", B=2, L=700, C=128, K=15, lens=(2, 1), mul=256)]
TANH_ABS = 2.0 ** -20        # tanhf: a few ulps of a result <= 1, allowed on top of tau * m (as voc_cases.run_post)


# ------------------------------------------------------------------------------------------------------------------------------
# plans: what the cases launch and what the engine can launch
# ------------------------------------------------------------------------------------------------------------------------------
def valid_rows(c):
    return [u * c["mul"] for u in c["units"]]


def case_pairs(lib):
    """({(layer, variant)} of every launch of the cases, {(layer, batch variant, batch-1 variant)} of every item of a batch)."""
    keys, pairs = set(), set()
    for c in conv_cases():
        valid = valid_rows(c)
        p = am_plans.conv1d_plan(lib, c["B"], max(valid), c["Cin"], c["Cout"], c["K"], c["dil"])["key"]
        keys.add((c["layer"], p))
        if c["B"] > 1:
            for n in valid:
                p1 = am_plans.conv1d_plan(lib, 1, n, c["Cin"], c["Cout"], c["K"], c["dil"])["key"]
                keys.add((c["layer"], p1))
                pairs.add((c["layer"], p, p1))
    return keys, pairs


def engine_workloads():
    """(B, phonemes per item, frames per item) of the corpus's batches at B in ENGINE_B."""
    from emotivoice_b200 import synth
    for B in ENGINE_B:
        lens = synth.corpus_lengths(B)
        for r in FRAMES_PER_PHONEME:
            yield B, lens, [max(1, int(r * n)) for n in lens]


def _am_records(B, T, F):
    return [r for r in am_plans.am_layers(B, T, F, "fp32_ffma", 1) if isinstance(r, dict)]


def engine_pairs(lib):
    """({(layer, variant)}, {(layer, batch variant, batch-1 variant)}) the engine launches in "fp32_ffma" over engine_workloads():
    the acoustic model's layers (kinds of am_plans.am_layers) and the vocoder's (kinds of voc_plans.ffma_layers)."""
    keys, pairs = set(), set()
    plan = lambda r: am_plans.conv1d_plan(lib, r["B"], r["L"], r["Cin"], r["Cout"], r["K"], r.get("dil", 1))["key"]
    for B, lens, frames in engine_workloads():
        batch = [(r["kind"], plan(r)) for r in _am_records(B, max(lens), max(frames))]
        batch += [(r["kind"], plan(r)) for r in voc_plans.ffma_layers(B, max(frames))]
        keys.update(batch)
        if B == 1:
            continue
        for n, f in zip(lens, frames):
            one = [(r["kind"], plan(r)) for r in _am_records(1, n, f)] + [(r["kind"], plan(r)) for r in voc_plans.ffma_layers(1, f)]
            keys.update(one)
            pairs.update((k, pb, p1) for (k, pb), (_, p1) in zip(batch, one))
    return keys, pairs


# ------------------------------------------------------------------------------------------------------------------------------
# running one case (on the GPU)
# ------------------------------------------------------------------------------------------------------------------------------
def _bits(t):
    import torch
    return t.contiguous().view(torch.int32)


def _nan_past(t, valid):
    t = t.clone()
    for b, n in enumerate(valid):
        t[b, n:] = float("nan")
    return t


def _zeros_past(t, valid):
    return all(bool((t[b, n:] == 0).all()) for b, n in enumerate(valid))


def _ptr(t):
    return None if t is None else t.data_ptr()


def run_conv(lib, dev, c, seed):
    """One conv1d_tm case -> a row: rc, the plan, err/m, rel_max, finite, pad_zero and the bitwise checks."""
    import torch
    import am_ref
    import voc_ref
    st = torch.cuda.current_stream().cuda_stream
    B, Cin, Cout, K, dil, rate, mul = c["B"], c["Cin"], c["Cout"], c["K"], c["dil"], c["rate"], c["mul"]
    valid = valid_rows(c)
    L = max(valid)
    acc, res_kind = c["acc"], c["res"]
    inplace = res_kind == "inplace"
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, Cin, generator=g)
    x = _nan_past(torch.nn.functional.gelu(x) if c["gelu_in"] else x, valid)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    bias = torch.randn(B if c["per_item"] else 1, Cout, generator=g)
    res = _nan_past(torch.randn(B, L, Cout, generator=g), valid) if res_kind else None
    prev = _nan_past(torch.randn(B, L, Cout, generator=g), valid) if acc else None
    init = res if inplace else (prev if acc else torch.full((B, L, Cout), float("nan")))
    xd, wd, bd = x.to(dev), w.to(dev), bias.to(dev)
    lens_d = torch.tensor(c["units"], dtype=torch.int32, device=dev) if c["lens"] else None
    bias_bs = Cout if c["per_item"] else 0

    def launch(x_, res_, out_, B_, L_, lens_, bias_):
        return lib.ev_op_conv1d(_ptr(x_), _ptr(wd), _ptr(bias_), bias_bs, _ptr(res_), _ptr(out_), B_, L_, Cin, Cout, K, dil, _ptr(lens_), mul,
                                c["act"], SLOPE, c["out_act"], acc, 3.0, st)

    plan = am_plans.conv1d_plan(lib, B, L, Cin, Cout, K, dil)
    row = dict(layer=c["layer"], variant=list(plan["key"][1:]), B=B, L=L, lens=c["units"], lens_mul=mul)
    out = init.to(dev)
    rd = out if inplace else (res.to(dev) if res is not None else None)
    rc = launch(xd, rd, out, B, L, lens_d, bd)
    torch.cuda.synchronize()
    row["rc"] = rc
    if rc != 0:
        return dict(row, err=lib.ev_last_error().decode(errors="replace"))
    got = out.cpu()
    row["pad_zero"] = _zeros_past(got, valid)
    if res_kind and acc == 0:
        # the other way to pass the residual -- a separate buffer where the engine adds it in place (out == res), in place where it
        # reads another buffer -- gives the same bits
        if inplace:
            o2 = torch.full((B, L, Cout), float("nan"), device=dev)
            rc2 = launch(xd, res.to(dev), o2, B, L, lens_d, bd)
        else:
            o2 = res.to(dev)
            rc2 = launch(xd, o2, o2, B, L, lens_d, bd)
        torch.cuda.synchronize()
        g2 = o2.cpu()
        row["bitwise_inplace_vs_separate_res"] = rc2 == 0 and all(_bits(got[b, :n]).equal(_bits(g2[b, :n])) for b, n in enumerate(valid)) \
            and _zeros_past(g2, valid)
    acc_chk = am_cases.Acc(1, voc_ref.REL_MAX[1])
    ov = got.view(B, L * rate, Cout // rate)
    for b, n in enumerate(valid):
        wins = voc_ref.windows(n, plan["BM"]) if n > 1024 else [(0, n)]
        for r0, r1 in wins:
            if c["family"] == "am":
                y64, m = am_ref.conv_ref(x[b], w, bias[b if c["per_item"] else 0], None if res is None else res[b], n, c["out_act"], r0, r1)
            else:
                y64, m = voc_ref.conv_ref(x[b], w, bias[0], None if res is None else res[b], None if prev is None else prev[b], n, r0, r1,
                                          dil, rate, bool(c["act"]), acc, 3.0)
            acc_chk.add(ov[b, r0 * rate:r1 * rate], y64, m)
    row.update(acc_chk.row())
    if B > 1:
        # every item alone (batch 1, no lens): the same bits, whatever variant the launcher picks for it
        same, pairs = True, []
        for b, n in enumerate(valid):
            x1 = xd[b:b + 1, :n].contiguous()
            o1 = init[b:b + 1, :n].contiguous().to(dev)
            r1 = o1 if inplace else (res[b:b + 1, :n].contiguous().to(dev) if res is not None else None)
            b1 = bd[b:b + 1].contiguous() if c["per_item"] else bd
            rc1 = launch(x1, r1, o1, 1, n, None, b1)
            torch.cuda.synchronize()
            same = same and rc1 == 0 and _bits(o1.cpu()[0]).equal(_bits(got[b, :n]))
            pairs.append(list(am_plans.conv1d_plan(lib, 1, n, Cin, Cout, K, dil)["key"][1:]))
        row["bitwise_item_vs_batch1"] = same
        row["item_variants"] = pairs
    return row


def run_post(lib, dev, c, seed):
    """One conv_post case -> a row: err/m against voc_ref.post_ref, pad_zero, and the bits of the granule-planar kernel on the same
    values (ev_op_to_gp + ev_op_conv_post_gp at bf16 = 0)."""
    import torch
    import voc_ref
    st = torch.cuda.current_stream().cuda_stream
    B, L, C, K, mul, lens = c["B"], c["L"], c["C"], c["K"], c["mul"], c["lens"]
    valid = [L] * B if lens is None else [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    x = _nan_past(torch.randn(B, L, C, generator=g) * 2, valid)
    w = torch.randn(K, C, generator=g) * (0.1 * math.sqrt(224.0 / (K * C)))
    bias = torch.randn(1, generator=g)
    xd, wd, bd = x.to(dev), w.to(dev), bias.to(dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev) if lens is not None else None
    wav = torch.full((B, L), float("nan"), device=dev)
    rc = lib.ev_op_conv_post(_ptr(xd), _ptr(wd), _ptr(bd), _ptr(lens_d), mul, B, L, C, K, 0.01, _ptr(wav), st)
    torch.cuda.synchronize()
    row = dict(rc=rc, B=B, L=L, C=C, K=K, lens=lens)
    if rc != 0:
        return dict(row, err=lib.ev_last_error().decode(errors="replace"))
    got = wav.cpu()
    err_m, num, den, fin = 0.0, 0.0, 0.0, True
    for b, n in enumerate(valid):
        y64, m = voc_ref.post_ref(x[b], w, bias, n)
        y = got[b, :n]
        fin = fin and bool(torch.isfinite(y).all())
        d = (y.double() - y64).abs()
        err_m = max(err_m, float(((d - TANH_ABS) / m).max()) if fin else float("inf"))
        num, den = max(num, float(d.max())), max(den, float(y64.abs().max()))
    rel = num / den if den > 0 and fin else float("inf")
    row.update(err_m=err_m, rel_max=rel, finite=fin, pad_zero=_zeros_past(got, valid),
               bound_ok=bool(fin and err_m <= voc_ref.TAU[1] and rel <= voc_ref.REL_MAX[1]))
    xg = torch.empty((B, C // 4, L, 4), device=dev)
    wav2 = torch.full((B, L), float("nan"), device=dev)
    rc1 = lib.ev_op_to_gp(_ptr(xd), L * C, C, 1, _ptr(xg), B, L, C, 0, st)
    rc2 = lib.ev_op_conv_post_gp(_ptr(xg), 0, _ptr(wd), _ptr(bd), _ptr(lens_d), mul, B, L, C, K, 0.01, _ptr(wav2), st)
    torch.cuda.synchronize()
    row["bitwise_vs_conv_post_gp"] = rc1 == 0 and rc2 == 0 and _bits(wav2.cpu()).equal(_bits(got))
    return row
