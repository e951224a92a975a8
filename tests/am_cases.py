"""Operator cases of the acoustic model's and the style encoder's tensor-core kernels, and the child process that runs them on
the GPU.

    python tests/am_cases.py <family>

runs one kernel family ("tc": the acoustic model's conv1d_tc + splitk_reduce through ev_op_conv1d_tc_ks; "attn": attention_tc;
"style": the style encoder's GEMMs, the same kernels at its layers) and prints one JSON row per case: the plan, the item
lengths, the largest per-element error relative to the fp64 bound (am_ref), the bitwise cross-checks and whether rows past each
item came out as the contract says.  tests/test_am_kernels_gpu.py and tests/test_style_kernels_gpu.py run each family once in
its own process under a timeout and assert every row.

Inputs hold NaN in every row at or past an item's length: a kernel that read such a row, even to mask it afterwards, would turn
a valid output into NaN (0 * NaN); residual rows there hold NaN too.  Outputs are prefilled with NaN (with the residual where
the engine adds it in place), and the split-K scratch with NaN as well.  Valid conv rows must be finite and within the bound;
conv rows at or past an item's length must be exact zeros (conv1d_tc's epilogue and splitk_reduce_store).  Attention rows below
klen must be finite and within the bound.

The longest fp32 chain of the style cases: a 3xTF32 ffn2 slice of BERT-base at C_in = 3072 and S = 4 is 768 products, so the
worst-case fp32 accumulation error is 767 * 2^-24 ~ 2^-14.4 of m, plus ~2^-21 of 3xTF32 operand error: under tau = 2^-14 of
MODE 1, with little margin in that worst case (typical rounding errors grow like the square root of the chain, far below it).
"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(1, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))      # emotivoice_b200 (the style layer shapes)

import am_plans  # noqa: E402
import style_plans  # noqa: E402
import voc_cases  # noqa: E402

H, N_MELS = 384, 80
ACT_NONE, ACT_RELU, ACT_GELU = am_plans.ACT_NONE, am_plans.ACT_RELU, am_plans.ACT_GELU
# kind -> (Cin, Cout, K, out_act, residual, per-item bias, input is a GELU output): the layers of am_plans.am_layers.  residual:
# None, "inplace" (the engine adds it in place: out == res) or "separate" (read from another buffer than the output)
KINDS = {"qkv": (H, 3 * H, 1, ACT_NONE, None, False, False),
         "wo": (H, H, 1, ACT_NONE, "inplace", False, False),
         "ffn1": (H, 4 * H, 3, ACT_GELU, None, False, False),
         "ffn2": (4 * H, H, 3, ACT_NONE, "inplace", False, False),
         "cond.wx": (H, H, 1, ACT_NONE, None, True, False),
         "pred": (H, H, 3, ACT_RELU, None, False, False),
         "to_mel": (H, N_MELS, 1, ACT_NONE, None, False, False)}
# every layer an operator case can run: the acoustic model's and the style encoder's of both configurations
LAYERS = dict(KINDS)
for _cfg in style_plans.CONFIGS:
    LAYERS.update(style_plans.layer_table(_cfg))
PREFIX = [("qkv", am_plans.ENC_SPLITS["qkv"]), ("wo", am_plans.ENC_SPLITS["wo"]), ("ffn1", am_plans.ENC_SPLITS["ffn1"]),
          ("ffn2", am_plans.ENC_SPLITS["ffn2"]), ("cond.wx", am_plans.COND_SPLIT), ("pred", am_plans.PRED_SPLIT)]
DECODER = [("qkv", am_plans.DEC_SPLITS["qkv"]), ("wo", am_plans.DEC_SPLITS["wo"]), ("ffn1", am_plans.DEC_SPLITS["ffn1"]),
           ("ffn2", am_plans.DEC_SPLITS["ffn2"]), ("to_mel", am_plans.MEL_SPLIT)]
DEC_MODES = (3, 0, 2)          # bf16x3 ("fp32"), 1xTF32 ("tf32"), bf16 ("bf16")
# batch-1 lengths per layer: one per N tile width the engine picks for it at B = 1 (BN halves while the launch has fewer than
# 24 output tiles: phonemes 12-200, frames 58-2148); the batch-32 cases have BN = 128 everywhere (80 for to_mel)
PREFIX_L1 = {"qkv": (100, 200), "wo": (100,), "ffn1": (100, 200), "ffn2": (100,), "cond.wx": (100,), "pred": (100,)}
DEC_L1 = {"qkv": (58, 249, 537), "wo": (58, 537, 1100), "ffn1": (58, 537), "ffn2": (58, 537, 1100), "to_mel": (537,)}
PREFIX_L32, DEC_L32 = 200, 200
EDGE_LENS = (1, 127, 128, 129)
B32 = 32


def ragged_lens(L, B=B32, seed=0):
    """Item lengths of the batch-32 case: L, the tile edges 1 / 127 / 128 / 129 (1: an item inside one conv halo), 63 / 64 / 65,
    2, and the rest spread over [1, L]."""
    import random
    rnd = random.Random(seed)
    head = [L, *EDGE_LENS, 63, 64, 65, 2]
    return [min(L, n) for n in head] + [rnd.randint(1, L) for _ in range(B - len(head))]


def _tc_cases():
    cs = []
    for mode, layers, l1, l32 in [(am_plans.PREFIX_MODE, PREFIX, PREFIX_L1, PREFIX_L32)] + [(m, DECODER, DEC_L1, DEC_L32) for m in DEC_MODES]:
        for kind, S in layers:
            for L in l1[kind]:
                cs.append(dict(name="%s_S%d_B1_L%d" % (kind.replace(".", ""), S, L), kind=kind, S=S, mode=mode, B=1, L=L))
            cs.append(dict(name="%s_S%d_B32_L%d" % (kind.replace(".", ""), S, l32), kind=kind, S=S, mode=mode, B=B32, L=l32))
    return cs


def _attn_cases():
    cs = [dict(name="enc_L%d" % L, B=1, L=L, lens=[L]) for L in (12, 50, 100, 200)]
    cs += [dict(name="dec_L%d" % L, B=1, L=L, lens=None) for L in (64, 129, 537, 2148)]
    cs += [dict(name="ragged_B32_L300", B=B32, L=300, lens=[300, 1, 63, 64, 65, 127, 128, 129] + ragged_lens(300, seed=5)[8:])]
    cs += [dict(name="lazy_rescale", B=2, L=400, lens=[400, 333], lazy=True)]
    return cs


# The style encoder's GEMMs (style_plans): the four layers of both configurations in MODE 1 ("fp32") and MODE 0 ("tf32"), each at
# the engine's own S, bias, GELU and residual.  Batch-1 lengths: every N tile width the planner picks at B = 1 and the 128-row
# edges next to each change (BERT-base: wo and ffn2 take BN = 32 up to 128 tokens, 64 for 129-384 and 128 above; qkv 64 up to
# 128 tokens and 128 above; ffn1 always 128.  The small model stays at BN = 32 at B = 1 over its 128 positions).  Ragged
# batches: items on the edges first, then random lengths; they run at BN = 128, except the small model's batch of 8 (wo, ffn2
# at BN = 64) and of 2 (qkv, ffn1 at BN = 64; wo, ffn2 at 32).
STYLE_L1 = {"base": (1, 20, 128, 129, 384, 385, 512), "small": (1, 20, 127, 128)}
STYLE_RAGGED = {"base": ((32, (64, 1, 2, 31, 32, 33, 63)), (8, (512, 1, 127, 128, 129, 255, 256, 257))),
                "small": ((32, (64, 1, 2, 31, 32, 33, 63)), (8, (128, 1, 127, 2, 63, 64, 65)), (2, (128, 1)))}


def style_lens(B, head, seed):
    """Item lengths of a ragged style case: `head` (the longest first), then random lengths in [1, head[0]]."""
    import random
    rnd = random.Random(seed)
    return list(head) + [rnd.randint(1, head[0]) for _ in range(B - len(head))]


def _style_cases():
    cs = []
    for cfg in style_plans.CONFIGS:
        for mode in (1, 0):
            for kind in style_plans.KINDS:
                S, k = style_plans.SPLITS[kind], style_plans.kind_name(cfg, kind)
                for L in STYLE_L1[cfg]:
                    cs.append(dict(name="%s_%s_S%d_B1_L%d" % (cfg, kind, S, L), kind=k, S=S, mode=mode, B=1, L=L))
                for B, head in STYLE_RAGGED[cfg]:
                    cs.append(dict(name="%s_%s_S%d_B%d_L%d" % (cfg, kind, S, B, head[0]), kind=k, S=S, mode=mode, B=B, L=head[0],
                                   lens=style_lens(B, head, seed=B + head[0]), edges=len(head)))
    return cs


FAMILIES = {"tc": _tc_cases, "attn": _attn_cases, "style": _style_cases}
MODES = {"tc": None, "attn": (1, 0), "style": None}


def case_ids(family):
    if MODES[family] is None:
        return ["%s-%s-m%d" % (family, c["name"], c["mode"]) for c in FAMILIES[family]()]
    return ["%s-%s-m%d" % (family, c["name"], m) for c in FAMILIES[family]() for m in MODES[family]]


def case_plans(lib, family="tc"):
    """{(layer kind, plan key)} of every case's launch of a GEMM family ("tc" or "style"; host-only), for the coverage tests."""
    keys = set()
    for c in FAMILIES[family]():
        Cin, Cout, K = LAYERS[c["kind"]][:3]
        keys.add((c["kind"], am_plans.tc_plan(lib, c["B"], c["L"], Cin, Cout, K, c["mode"], c["S"])["key"]))
    return keys


# ------------------------------------------------------------------------------------------------------------------------------
# child process
# ------------------------------------------------------------------------------------------------------------------------------
def _nan_past(t, valid):
    t = t.clone()
    for b, n in enumerate(valid):
        t[b, n:] = float("nan")
    return t


def _valid_equal(a, b, valid):
    bits = voc_cases._bits
    return all(bits(a[i, :n].contiguous()).equal(bits(b[i, :n].contiguous())) for i, n in enumerate(valid))


def _zeros_past(t, valid):
    return all(bool((t[i, n:] == 0).all()) and not bool(t[i, n:].isnan().any()) for i, n in enumerate(valid))


class Acc:
    """The per-element check accumulated over a case's items."""
    def __init__(self, mode, rel_lim):
        self.mode, self.rel_lim, self.err_m, self.num, self.den, self.finite = mode, rel_lim, 0.0, 0.0, 0.0, True

    def add(self, y, y64, m):
        import torch
        import voc_ref
        self.finite = self.finite and bool(torch.isfinite(y).all())
        e = voc_ref.bound_excess(y, y64, m, voc_ref.TAU[self.mode])
        if e.numel():
            self.err_m = max(self.err_m, float(e.max()))
            self.num = max(self.num, float((y.double() - y64).abs().max()))
            self.den = max(self.den, float(y64.abs().max()))

    def row(self):
        import voc_ref
        rel = self.num / self.den if self.den > 0 else 0.0
        if not (math.isfinite(self.err_m) and math.isfinite(rel)):
            rel = float("inf")
        ok = self.finite and self.err_m <= voc_ref.TAU[self.mode] and rel <= self.rel_lim
        return dict(err_m=self.err_m, rel_max=rel, finite=self.finite, bound_ok=bool(ok))


def run_tc(R, c, seed):
    import torch
    import am_ref
    lib, dev = R.lib, R.dev
    B, L, mode, S = c["B"], c["L"], c["mode"], c["S"]
    Cin, Cout, K, oact, res_kind, per_item, gelu_in = LAYERS[c["kind"]]
    inplace = res_kind == "inplace"
    pl = am_plans.tc_plan(lib, B, L, Cin, Cout, K, mode, S)
    valid = c.get("lens") or (ragged_lens(L, B, seed) if B > 1 else [L])
    row = dict(kind=c["kind"], plan=list(pl["key"]), B=B, L=L, lens=valid)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, Cin, generator=g)          # LayerNorm-like rows; a GELU output where the layer reads one
    x = _nan_past(torch.nn.functional.gelu(x) if gelu_in else x, valid)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    bias = torch.randn(B if per_item else 1, Cout, generator=g)
    res = _nan_past(torch.randn(B, L, Cout, generator=g), valid) if res_kind else None
    xd, wd, bd = x.to(dev), voc_cases._pack(mode)(w).to(dev), bias.to(dev)
    lens_d = torch.tensor(valid, dtype=torch.int32, device=dev) if B > 1 else None
    bias_bs = Cout if per_item else 0

    def launch(x_, res_, out_, B_, L_, lens_):
        ws = torch.full((pl["S"] * B_ * L_ * Cout,), float("nan"), device=dev) if S > 1 else None
        R.keep.append(ws)
        return lib.ev_op_conv1d_tc_ks(R.ptr(x_), R.ptr(wd), mode, R.ptr(bd), bias_bs, R.ptr(res_), R.ptr(out_), B_, L_, Cin, Cout, K, 1,
                                      R.ptr(lens_), 1, 0, 0.0, oact, 0, 1.0, S, R.ptr(ws), 0 if ws is None else ws.numel(), R.st)

    def run_once(inplace_res):
        if inplace_res:
            out = res.to(dev)
            rc = launch(xd, out, out, B, L, lens_d)
        else:
            out = torch.full((B, L, Cout), float("nan"), device=dev)
            rd = res.to(dev) if res is not None else None
            R.keep.append(rd)
            rc = launch(xd, rd, out, B, L, lens_d)
        R.keep.append(out)
        return rc, out

    rc, out1 = run_once(inplace)
    rc2, out2 = run_once(inplace)
    torch.cuda.synchronize()
    row["rc"] = rc
    if rc != 0 or rc2 != 0:
        return dict(row, rc=rc or rc2, err=R.err())
    got = out1.cpu()
    row["bitwise_two_runs"] = _valid_equal(got, out2.cpu(), valid) and _zeros_past(out2.cpu(), valid)
    row["pad_zero"] = _zeros_past(got, valid)
    if inplace:
        rc3, out3 = run_once(False)
        torch.cuda.synchronize()
        row["bitwise_inplace_vs_out_of_place"] = rc3 == 0 and _valid_equal(got, out3.cpu(), valid) and _zeros_past(out3.cpu(), valid)
    acc = Acc(mode, am_ref.REL_MAX[mode])
    for b, n in enumerate(valid):
        y64, m = am_ref.conv_ref(x[b], w, bias[b if per_item else 0], None if res is None else res[b], n, oact)
        acc.add(got[b, :n], y64, m)
    row.update(acc.row())
    if B > 1:
        # an item of the ragged batch == its own batch-1 launch (another BN and other rings, the same KBG and slices)
        same = True
        for b, n in enumerate(valid):
            if b >= c["edges"] if "edges" in c else (n not in EDGE_LENS + (L,) or valid.index(n) != b):
                continue
            x1 = xd[b:b + 1, :n].contiguous()
            o1 = res[b:b + 1, :n].contiguous().to(dev) if inplace else torch.full((1, n, Cout), float("nan"), device=dev)
            r1 = o1 if inplace else (res[b:b + 1, :n].contiguous().to(dev) if res_kind else None)
            if per_item:
                b1 = bd[b:b + 1].contiguous()
            R.keep += [x1, o1, r1]
            ws = torch.full((pl["S"] * n * Cout,), float("nan"), device=dev) if S > 1 else None
            R.keep.append(ws)
            rc1 = lib.ev_op_conv1d_tc_ks(R.ptr(x1), R.ptr(wd), mode, R.ptr(b1 if per_item else bd), bias_bs, R.ptr(r1),
                                         R.ptr(o1), 1, n, Cin, Cout, K, 1, None, 1, 0, 0.0, oact, 0, 1.0, S, R.ptr(ws),
                                         0 if ws is None else ws.numel(), R.st)
            torch.cuda.synchronize()
            same = same and rc1 == 0 and voc_cases._bits(o1.cpu()[0]).equal(voc_cases._bits(got[b, :n].contiguous()))
        row["bitwise_item_vs_batch1"] = same
    return row


def run_attn(R, c, mode, seed):
    import torch
    import am_ref
    import voc_ref
    lib, dev = R.lib, R.dev
    B, L, heads = c["B"], c["L"], 8
    lens = c["lens"]
    valid = lens if lens is not None else [L] * B
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, L, 3 * H, generator=g)
    rel_lim = am_ref.ATTN_REL_MAX[mode]
    if c.get("lazy"):          # test_attention_tc_lazy_rescale_path's construction: key tiles growing past the rescale threshold
        qkv[:, :, H:2 * H] *= (1.0 + 2.5 * (torch.arange(L) // 64).float())[None, :, None]
        qkv[:, 1::3, :H] *= 0.05
        rel_lim = am_ref.ATTN_REL_MAX_LARGE_SCORES[mode]
    qkv = _nan_past(qkv, valid)
    qd = qkv.to(dev)
    ld = torch.tensor(lens, dtype=torch.int32, device=dev) if lens is not None else None
    out = torch.full((B, L, H), float("nan"), device=dev)
    out2 = torch.full((B, L, H), float("nan"), device=dev)
    rc = lib.ev_op_attention_tc(R.ptr(qd), R.ptr(ld), R.ptr(out), B, L, H, heads, mode, R.st)
    rc2 = lib.ev_op_attention_tc(R.ptr(qd), R.ptr(ld), R.ptr(out2), B, L, H, heads, mode, R.st)
    torch.cuda.synchronize()
    row = dict(B=B, L=L, lens=lens, rc=rc or rc2)
    if rc != 0 or rc2 != 0:
        return dict(row, err=R.err())
    got = out.cpu()
    row["bitwise_two_runs"] = _valid_equal(got, out2.cpu(), valid)
    acc = Acc(mode, rel_lim)
    for b, n in enumerate(valid):
        rows = torch.cat([torch.arange(a, e) for a, e in voc_ref.windows(n, 128)]) if n > 1024 else torch.arange(n)
        y64, m = am_ref.attn_ref(qkv[b], n, heads, rows)
        acc.add(got[b, rows], y64, m)
    row.update(acc.row())
    if B > 1:
        same = True
        done = set()
        for b, n in enumerate(valid):
            if n in done:
                continue
            done.add(n)
            q1 = qd[b:b + 1, :n].contiguous()
            o1 = torch.full((1, n, H), float("nan"), device=dev)
            R.keep += [q1, o1]
            rc1 = lib.ev_op_attention_tc(R.ptr(q1), None, R.ptr(o1), 1, n, H, heads, mode, R.st)
            torch.cuda.synchronize()
            same = same and rc1 == 0 and voc_cases._bits(o1.cpu()[0]).equal(voc_cases._bits(got[b, :n].contiguous()))
        row["bitwise_item_vs_batch1"] = same
    return row


def main(family):
    lib = voc_cases._setup()
    import torch
    R = voc_cases.Runner(lib)
    if family in ("tc", "style"):
        for i, c in enumerate(FAMILIES[family]()):
            cid = "%s-%s-m%d" % (family, c["name"], c["mode"])
            try:
                row = run_tc(R, c, 1000 * i + 7)
            except Exception as e:      # a Python-side error in one case must not hide the others' rows
                row = dict(exception="%s: %s" % (type(e).__name__, e))
            print(json.dumps(dict(id=cid, mode=c["mode"], **row)), flush=True)
            R.keep.clear()
            torch.cuda.empty_cache()
        return
    for i, c in enumerate(_attn_cases()):
        for mode in MODES["attn"]:
            cid = "attn-%s-m%d" % (c["name"], mode)
            try:
                row = run_attn(R, c, mode, 100 * i + mode + 3)
            except Exception as e:
                row = dict(exception="%s: %s" % (type(e).__name__, e))
            print(json.dumps(dict(id=cid, mode=mode, **row)), flush=True)
            R.keep.clear()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main(sys.argv[1])
