"""Operator cases of the vocoder's granule-planar kernels, and the child process that runs them on the GPU.

    python tests/voc_cases.py <family>

runs one kernel family and prints one JSON row per case: the plan the kernel ran with, the item lengths, the largest
per-element error relative to the fp64 bound (voc_ref), the bitwise cross-checks and whether rows past each item were left
alone.  tests/test_voc_kernels_gpu.py runs each family once in its own process under a timeout (a deadlocked pipeline then
ends that child, not the suite) and asserts every row.

Inputs hold NaN in every row past an item's valid length: the kernels must treat those rows as zero padding without reading
them.  Outputs are prefilled with NaN (or, for the accumulate epilogues, with the previous values in the valid rows); rows past
the valid length must keep their bits.
"""
import ctypes
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODES = (0, 1, 2, 3)
CONV_L = {256: 1800, 128: 3000, 64: 6000, 32: 12000}


def _conv_cases():
    cs = [dict(name="pre", B=2, L=700, Cin=80, Cout=512, K=7, dil=1, rate=1, act=0, res=0, acc=0),
          dict(name="ups0", B=2, L=300, Cin=512, Cout=2048, K=3, dil=1, rate=8, act=1, res=0, acc=0),
          dict(name="ups1", B=2, L=1500, Cin=256, Cout=1024, K=3, dil=1, rate=8, act=1, res=0, acc=0),
          dict(name="ups2", B=3, L=6000, Cin=128, Cout=128, K=3, dil=1, rate=2, act=1, res=0, acc=0),
          dict(name="ups3", B=2, L=20000, Cin=64, Cout=64, K=3, dil=1, rate=2, act=1, res=0, acc=0)]
    for C in (256, 128, 64, 32):
        for K in (3, 7, 11):
            for d in (1, 3, 5):
                cs.append(dict(name="c1_C%d_k%d_d%d" % (C, K, d), B=2, L=CONV_L[C], Cin=C, Cout=C, K=K, dil=d, rate=1, act=1, res=0, acc=0))
            cs.append(dict(name="c2_C%d_k%d" % (C, K), B=2, L=CONV_L[C], Cin=C, Cout=C, K=K, dil=1, rate=1, act=1, res=1, acc={3: 0, 7: 1, 11: 2}[K]))
    # long launches: four accumulators per tile, persistent CTAs walking several tiles, large-batch tile shapes
    cs += [dict(name="long_C32_k11_d5", B=3, L=70000, Cin=32, Cout=32, K=11, dil=5, rate=1, act=1, res=1, acc=2),
           dict(name="long_C64_k11_d3", B=4, L=40000, Cin=64, Cout=64, K=11, dil=3, rate=1, act=1, res=0, acc=0),
           dict(name="long_C128_k11", B=1, L=34368, Cin=128, Cout=128, K=11, dil=1, rate=1, act=1, res=1, acc=1),
           dict(name="long_C256_k7_d3", B=4, L=16000, Cin=256, Cout=256, K=7, dil=3, rate=1, act=1, res=0, acc=0),
           dict(name="long_ups0", B=8, L=2000, Cin=512, Cout=2048, K=3, dil=1, rate=8, act=1, res=0, acc=0),
           dict(name="long_ups1", B=8, L=8000, Cin=256, Cout=1024, K=3, dil=1, rate=8, act=1, res=0, acc=0),
           dict(name="long_pre", B=32, L=1100, Cin=80, Cout=512, K=7, dil=1, rate=1, act=0, res=0, acc=0)]
    # batch-1 shapes of very short utterances (F = 1 and 150 frames): one- and two-accumulator tiles, items shorter than the halo
    cs += [dict(name="ups3_F1", B=1, L=128, Cin=64, Cout=64, K=3, dil=1, rate=2, act=1, res=0, acc=0),
           dict(name="ups3_F150", B=1, L=19200, Cin=64, Cout=64, K=3, dil=1, rate=2, act=1, res=0, acc=0),
           dict(name="c1_C32_k11_d5_F1", B=1, L=256, Cin=32, Cout=32, K=11, dil=5, rate=1, act=1, res=0, acc=0)]
    return cs


def _pair_cases():
    cs = []
    for C, L in ((128, 4000), (64, 9000), (32, 20000)):
        for K in (3, 7, 11):
            for d in (1, 3, 5):
                cs.append(dict(name="C%d_k%d_d%d" % (C, K, d), B=3, L=L, C=C, K=K, dil=d, acc=(K + d) % 3))
    cs += [dict(name="long_C32_k7_d3", B=3, L=70000, C=32, K=7, dil=3, acc=1),
           dict(name="long_C64_k11_d5", B=4, L=40000, C=64, K=11, dil=5, acc=2),
           dict(name="long_C128_k3_d1", B=8, L=20000, C=128, K=3, dil=1, acc=0),
           dict(name="C64_k7_d3_F300", B=1, L=38400, C=64, K=7, dil=3, acc=0)]
    return cs


def _group_cases():
    cs = []
    for C, B, L in ((256, 1, 4296), (128, 1, 8592), (64, 2, 6000), (32, 1, 12000)):
        cs.append(dict(name="c1_C%d" % C, B=B, L=L, C=C, Ks=(3, 7, 11), dils=(1, 3, 5), res=0))
        cs.append(dict(name="c2_C%d" % C, B=B, L=L, C=C, Ks=(11, 3, 7), dils=(1, 1, 1), res=1))
    cs += [dict(name="two_C64", B=3, L=900, C=64, Ks=(7, 3), dils=(3, 1), res=0),
           dict(name="c1_C128_d5", B=2, L=3000, C=128, Ks=(3, 7, 11), dils=(5, 5, 5), res=1),
           dict(name="long_C128", B=1, L=34368, C=128, Ks=(3, 7, 11), dils=(3, 3, 3), res=0),
           dict(name="c1_C32_F1", B=1, L=256, C=32, Ks=(3, 7, 11), dils=(1, 3, 5), res=0),
           dict(name="c2_C32_F1", B=1, L=256, C=32, Ks=(3, 7, 11), dils=(1, 1, 1), res=1),
           dict(name="c1_C32_F40", B=1, L=10240, C=32, Ks=(3, 7, 11), dils=(5, 5, 5), res=0),
           dict(name="c2_C32_B2_F40", B=2, L=10240, C=32, Ks=(11, 3, 7), dils=(1, 1, 1), res=1),
           dict(name="c1_C64_F150", B=1, L=19200, C=64, Ks=(3, 7, 11), dils=(1, 3, 5), res=0)]
    return cs


def _pair_group_cases():
    cs = []
    for C, B, L in ((128, 1, 8592), (64, 1, 17184), (32, 1, 34368), (64, 2, 20000), (32, 3, 20000)):
        for d in (1, 3, 5):
            cs.append(dict(name="C%d_B%d_d%d" % (C, B, d), B=B, L=L, C=C, Ks=(3, 7, 11), dils=(d, d, d)))
    cs += [dict(name="long_C64", B=1, L=68736, C=64, Ks=(3, 7, 11), dils=(1, 3, 5)),
           dict(name="long_C32", B=1, L=137472, C=32, Ks=(11, 3, 7), dils=(5, 5, 5)),
           dict(name="two_C64", B=3, L=20000, C=64, Ks=(7, 3), dils=(1, 1))]
    return cs


def _post_cases():
    return [dict(name="k7_B3", B=3, L=5003, C=32, K=7, lens=(20, 13, 1), mul=256, bf=bf) for bf in (0, 1)] + \
           [dict(name="k7_nolens", B=1, L=1001, C=32, K=7, lens=None, mul=1, bf=0),
            dict(name="k5_B2", B=2, L=3001, C=32, K=5, lens=(11, 3), mul=256, bf=0),
            dict(name="k5_B2", B=2, L=3001, C=32, K=5, lens=(11, 3), mul=256, bf=1)]


FAMILIES = {"conv": _conv_cases, "pair": _pair_cases, "group": _group_cases, "pair_group": _pair_group_cases, "post": _post_cases}


def case_ids(family):
    if family == "post":
        return ["post-%s-bf%d" % (c["name"], c["bf"]) for c in _post_cases()] + ["post-to_gp-bf0", "post-to_gp-bf1"]
    return ["%s-%s-m%d" % (family, c["name"], m) for c in FAMILIES[family]() for m in MODES]


def case_plans(lib, family):
    """The plan key every operator case of a family runs with (host-only), for the coverage test."""
    import voc_plans as vp
    keys = set()
    for c in FAMILIES[family]():
        for m in MODES:
            if family == "conv":
                p = vp.gp_plan(lib, c["B"], c["L"], c["Cin"], c["Cout"], c["K"], c["dil"], c["rate"], m)
            elif family == "pair":
                p = vp.pair_plan(lib, c["B"], c["L"], c["C"], c["K"], c["dil"], m)
            elif family == "group":
                p = vp.gp_group_plan(lib, c["Ks"], c["dils"], c["B"], c["L"], c["C"], c["C"], m)
            else:
                p = vp.pair_group_plan(lib, c["Ks"], c["dils"], c["B"], c["L"], c["C"], m)
            if p is not None:
                keys.add(p["key"])
    return keys


# ------------------------------------------------------------------------------------------------------------------------------
# lengths: valid lengths at tile edges
# ------------------------------------------------------------------------------------------------------------------------------
CONV_RESIDUES = (0, 1, 63, 64, 65, 127)


def pick_lens(B, L, tile, residues, mul, tiny=False):
    """Item lengths (in units of `mul` rows) so that item 0 is L rows long (capped), the next items end at k * tile + r for the
    given residues r (as long as possible, k >= 0), and, with tiny, the last item is one unit (mul rows) long."""
    out = [-(-L // mul)]
    ri = 0
    want = B - 1 - (1 if tiny else 0)
    frac = [0.8, 0.45, 0.2, 0.6, 0.3, 0.1, 0.7]
    while len(out) < 1 + want:
        r = residues[ri % len(residues)]
        top = int(L * frac[(len(out) - 1) % len(frac)])
        k = max(0, (top - r) // tile)
        n = None
        while k >= 0:
            cand = k * tile + r
            if 0 < cand <= L and cand % mul == 0:
                n = cand
                break
            k -= 1
        ri += 1
        if n is not None:
            out.append(n // mul)
        elif ri > 10 * len(residues):
            out.append(max(1, (top // mul)))
    if tiny:
        out.append(1)
    return out[:B]


def odd_mul(tile):
    for m in (3, 5, 7, 11, 13):
        if math.gcd(m, tile) == 1:
            return m
    return 1


# ------------------------------------------------------------------------------------------------------------------------------
# child process
# ------------------------------------------------------------------------------------------------------------------------------
def _setup():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch
    from emotivoice_b200 import _abi, build
    build.build(verbose=False)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _abi.load()


class Runner:
    def __init__(self, lib):
        import torch
        self.torch = torch
        self.lib = lib
        self.dev = torch.device("cuda:0")
        self.st = torch.cuda.current_stream().cuda_stream
        self.keep = []             # device tensors stay alive until the row is finished: no address is recycled mid-case

    def ptr(self, t):
        return None if t is None else t.data_ptr()

    def err(self):
        return self.lib.ev_last_error().decode(errors="replace")


def _bits(t):
    import torch
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _nan_past(t, valid):
    """Copy of (B, L, C) t with rows >= valid[b] set to NaN."""
    t = t.clone()
    for b, n in enumerate(valid):
        t[b, n:] = float("nan")
    return t


def _pack(mode):
    from emotivoice_b200 import packing
    return packing.to_tc16x2_layout if mode == 3 else (packing.to_tc16_layout if mode == 2 else packing.to_tc_layout)


def _stored(t, bf):
    """The values a GP tensor of t holds (bf16-rounded in the bf16-storage mode)."""
    from emotivoice_b200 import layout
    return layout.from_gp(layout.to_gp(t, bf)) if bf else t


def _pad_ok(got_gp, before_gp, valid):
    """Rows >= valid[b] of the GP output keep their bits."""
    for b, n in enumerate(valid):
        if not _bits(got_gp[b, :, n:]).equal(_bits(before_gp[b, :, n:])):
            return False
    return True


def _gp_valid_equal(a_gp, b_gp, valid):
    for b, n in enumerate(valid):
        if not _bits(a_gp[b, :, :n]).equal(_bits(b_gp[b, :, :n])):
            return False
    return True


class Acc:
    """Accumulates the per-element check over the windows of a row."""
    def __init__(self, mode):
        self.mode, self.err_m, self.rel_num, self.rel_den, self.finite = mode, 0.0, 0.0, 0.0, True

    def add(self, y, y64, m):
        import voc_ref
        e = voc_ref.bound_excess(y, y64, m, voc_ref.TAU[self.mode], bf16_out=self.mode == 2)
        if e.numel():
            self.err_m = max(self.err_m, float(e.max()))
            self.rel_num = max(self.rel_num, float((y.double() - y64).abs().max()))
            self.rel_den = max(self.rel_den, float(y64.abs().max()))

    def check_finite(self, y):
        import torch
        self.finite = self.finite and bool(torch.isfinite(y).all())

    def row(self):
        import voc_ref
        rel = self.rel_num / self.rel_den if self.rel_den > 0 else 0.0
        if not math.isfinite(self.err_m):
            rel = float("inf")
        ok = self.finite and self.err_m <= voc_ref.TAU[self.mode] and rel <= voc_ref.REL_MAX[self.mode]
        return dict(err_m=self.err_m, rel_max=rel, finite=self.finite, bound_ok=bool(ok))


def run_conv(R, c, mode, seed):
    import torch
    import voc_plans as vp
    import voc_ref
    from emotivoice_b200 import _abi, layout
    lib, dev = R.lib, R.dev
    B, L, Cin, Cout, K, dil, rate = c["B"], c["L"], c["Cin"], c["Cout"], c["K"], c["dil"], c["rate"]
    pl = vp.gp_plan(lib, B, L, Cin, Cout, K, dil, rate, mode)
    row = dict(plan=pl and list(pl["key"]), L=L)
    if pl is None:
        return dict(row, rc=-1, err=R.err())
    tile = 128 * pl["MT"]
    mul = odd_mul(tile)
    lens = pick_lens(B, L, tile, CONV_RESIDUES[seed % 6:] + CONV_RESIDUES[:seed % 6], mul, tiny=(B >= 3))
    valid = [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    coutR = Cout // rate
    x = _nan_past(torch.randn(B, L, Cin, generator=g), valid)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    bias = torch.randn(Cout, generator=g)
    vout = [n * rate for n in valid]
    res = _nan_past(torch.randn(B, L * rate, coutR, generator=g), vout) if c["res"] else None
    prev = torch.randn(B, L * rate, coutR, generator=g)
    init = prev.clone() if c["acc"] else torch.full_like(prev, float("nan"))
    init = _nan_past(init, vout)
    bf = mode == 2
    xg, wd, bd = layout.to_gp(x, bf).to(dev), _pack(mode)(w).to(dev), bias.to(dev)
    rg = layout.to_gp(res, bf).to(dev) if res is not None else None
    before = layout.to_gp(init, bf)
    og = before.to(dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    rc = lib.ev_op_conv1d_gp(R.ptr(xg), R.ptr(wd), mode, R.ptr(bd), R.ptr(rg), R.ptr(og), B, L, Cin, Cout, K, dil, rate, R.ptr(lens_d), mul,
                             _abi.ACT_LRELU if c["act"] else _abi.ACT_NONE, 0.1, c["acc"], 3.0, R.st)
    torch.cuda.synchronize()
    row.update(rc=rc, lens=lens, lens_mul=mul)
    if rc != 0:
        return dict(row, err=R.err())
    got_gp = og.cpu()
    got = layout.from_gp(got_gp)
    row["pad_untouched"] = _pad_ok(got_gp, before, vout)
    xs, rs, ps = _stored(x, bf), (_stored(res, bf) if res is not None else None), _stored(init, bf)
    acc = Acc(mode)
    for b, n in enumerate(valid):
        acc.check_finite(got[b, :n * rate])
        for r0, r1 in voc_ref.windows(n, tile):
            y64, m = voc_ref.conv_ref(xs[b], w, bias, None if rs is None else rs[b], ps[b], n, r0, r1, dil, rate, bool(c["act"]), c["acc"], 3.0)
            acc.add(got[b, r0 * rate:r1 * rate], y64, m)
    row.update(acc.row())
    if mode in (0, 1):
        # the time-major tensor-core kernel: same reduction order and roundings -> bitwise equal on the valid rows
        xt = torch.nan_to_num(x, nan=0.0).to(dev)
        ref = torch.nan_to_num(init, nan=0.0).reshape(B, L, Cout).contiguous().to(dev)
        rt = torch.nan_to_num(res, nan=0.0).reshape(B, L, Cout).contiguous().to(dev) if res is not None else None
        rc2 = lib.ev_op_conv1d_tc(R.ptr(xt), R.ptr(wd), mode, R.ptr(bd), 0, R.ptr(rt), R.ptr(ref), B, L, Cin, Cout, K, dil, R.ptr(lens_d), mul,
                                  _abi.ACT_LRELU if c["act"] else _abi.ACT_NONE, 0.1, _abi.ACT_NONE, c["acc"], 3.0, None, 0, R.st)
        torch.cuda.synchronize()
        ref = ref.cpu().reshape(B, L * rate, coutR)
        row["bitwise_vs_tc"] = rc2 == 0 and all(_bits(got[b, :n]).equal(_bits(ref[b, :n])) for b, n in enumerate(vout))
    return row


def _conv_launch(R, mode, x, w, bias, res, out, B, L, C, K, dil, lens_d, mul, acc=0, div=1.0):
    from emotivoice_b200 import _abi
    return R.lib.ev_op_conv1d_gp(R.ptr(x), R.ptr(w), mode, R.ptr(bias), R.ptr(res), R.ptr(out), B, L, C, C, K, dil, 1, R.ptr(lens_d), mul,
                                 _abi.ACT_LRELU, 0.1, acc, div, R.st)


def run_pair(R, c, mode, seed):
    import torch
    import voc_plans as vp
    import voc_ref
    from emotivoice_b200 import layout
    lib, dev = R.lib, R.dev
    B, L, C, K, dil, accm = c["B"], c["L"], c["C"], c["K"], c["dil"], c["acc"]
    pl = vp.pair_plan(lib, B, L, C, K, dil, mode)
    row = dict(plan=pl and list(pl["key"]), L=L)
    Rt = pl["R"] if pl else 128 - (K - 1)
    mul = odd_mul(Rt)
    lens = pick_lens(B, L, Rt, (0, 1, Rt - 1), mul, tiny=True)
    valid = [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    x = _nan_past(torch.randn(B, L, C, generator=g), valid)
    w1 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
    w2 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
    b1, b2 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    prev = torch.randn(B, L, C, generator=g)
    init = _nan_past(prev.clone() if accm else torch.full_like(prev, float("nan")), valid)
    bf = mode == 2
    xg = layout.to_gp(x, bf).to(dev)
    w1d, w2d, b1d, b2d = _pack(mode)(w1).to(dev), _pack(mode)(w2).to(dev), b1.to(dev), b2.to(dev)
    before = layout.to_gp(init, bf)
    out = before.to(dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    rc = lib.ev_op_resblock_gp(R.ptr(xg), R.ptr(w1d), R.ptr(b1d), R.ptr(w2d), R.ptr(b2d), mode, R.ptr(out), B, L, C, K, dil, R.ptr(lens_d), mul,
                               accm, 3.0, R.st)
    torch.cuda.synchronize()
    row.update(rc=rc, lens=lens, lens_mul=mul)
    if pl is None:
        # a shape the fused kernel does not take (the engine runs it as two launches): it must refuse, not compute
        return dict(row, unsupported=True)
    if rc != 0:
        return dict(row, err=R.err())
    got_gp = out.cpu()
    got = layout.from_gp(got_gp)
    row["pad_untouched"] = _pad_ok(got_gp, before, valid)
    xs, ps = _stored(x, bf), _stored(init, bf)
    rnd = (lambda t: t.float().to(torch.bfloat16).double()) if bf else None
    acc = Acc(mode)
    for b, n in enumerate(valid):
        acc.check_finite(got[b, :n])
        for r0, r1 in voc_ref.windows(n, Rt):
            y64, m = voc_ref.pair_ref(xs[b], w1, b1, w2, b2, ps[b], n, r0, r1, dil, accm, 3.0, xt_round=rnd)
            acc.add(got[b, r0:r1], y64, m)
    row.update(acc.row())
    # the two conv1d_gp launches it replaces: bitwise
    xt = torch.full_like(xg, float("nan"))
    ref = before.to(dev)
    rc1 = _conv_launch(R, mode, xg, w1d, b1d, None, xt, B, L, C, K, dil, lens_d, mul)
    rc2 = _conv_launch(R, mode, xt, w2d, b2d, xg, ref, B, L, C, K, 1, lens_d, mul, accm, 3.0)
    torch.cuda.synchronize()
    row["bitwise_vs_two_launches"] = rc1 == 0 and rc2 == 0 and _gp_valid_equal(got_gp, ref.cpu(), valid)
    return row


def _tab(R, ts):
    n = len(ts)
    return (ctypes.c_void_p * n)(*[R.ptr(t) for t in ts])


def run_group(R, c, mode, seed):
    import torch
    import voc_plans as vp
    import voc_ref
    from emotivoice_b200 import layout
    lib, dev = R.lib, R.dev
    B, L, C, Ks, dils, use_res = c["B"], c["L"], c["C"], list(c["Ks"]), list(c["dils"]), c["res"]
    n = len(Ks)
    pl = vp.gp_group_plan(lib, Ks, dils, B, L, C, C, mode)
    row = dict(plan=pl and list(pl["key"]), L=L)
    tile = 128 * pl["MT"] if pl else 128
    mul = odd_mul(tile)
    lens = pick_lens(B, L, tile, CONV_RESIDUES[seed % 6:] + CONV_RESIDUES[:seed % 6], mul, tiny=(B >= 3)) if B > 1 else [-(-L // mul)]
    if B == 1:           # one item: its length still lands on a tile edge
        r = CONV_RESIDUES[seed % 6]
        k = (L - r) // tile
        while k >= 0 and (k * tile + r == 0 or (k * tile + r) % mul):
            k -= 1
        lens = [max(1, (k * tile + r) // mul)]
    valid = [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    bf = mode == 2
    xs = [_nan_past(torch.randn(B, L, C, generator=g), valid) for _ in range(n)]
    ws = [torch.randn(K, C, C, generator=g) / math.sqrt(C * K) for K in Ks]
    bs = [torch.randn(C, generator=g) for _ in range(n)]
    # with use_res the output tensor is also the residual (the engine's in-place x_j += c2(...)): valid rows hold it
    init = [_nan_past(torch.randn(B, L, C, generator=g) if use_res else torch.full((B, L, C), float("nan")), valid) for _ in range(n)]
    wd = [_pack(mode)(w).to(dev) for w in ws]
    bd = [b_.to(dev) for b_ in bs]
    xg = [layout.to_gp(x, bf).to(dev) for x in xs]
    before = [layout.to_gp(t, bf) for t in init]
    grp = [t.to(dev) for t in before]
    solo = [t.to(dev) for t in before]
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    IA = ctypes.c_int * n
    from emotivoice_b200 import _abi
    rc = lib.ev_op_conv1d_gp_group(n, _tab(R, xg), _tab(R, wd), mode, _tab(R, bd), _tab(R, grp) if use_res else None, _tab(R, grp), IA(*Ks), IA(*dils),
                                   B, L, C, C, R.ptr(lens_d), mul, _abi.ACT_LRELU, 0.1, R.st)
    rcs = [_conv_launch(R, mode, xg[i], wd[i], bd[i], solo[i] if use_res else None, solo[i], B, L, C, Ks[i], dils[i], lens_d, mul) for i in range(n)]
    torch.cuda.synchronize()
    row.update(rc=rc, solo_rc=rcs, lens=lens, lens_mul=mul)
    if pl is None:
        # members whose own launches sum in different orders (K granules per stage) cannot share one: the launch must refuse
        return dict(row, unsupported=True)
    if rc != 0:
        return dict(row, err=R.err())
    acc = Acc(mode)
    eq, pad = not any(rcs), True
    for i in range(n):
        got_gp = grp[i].cpu()
        got = layout.from_gp(got_gp)
        pad = pad and _pad_ok(got_gp, before[i], valid)
        eq = eq and _gp_valid_equal(got_gp, solo[i].cpu(), valid)
        xs_i, rs_i = _stored(xs[i], bf), _stored(init[i], bf)
        for b, nv in enumerate(valid):
            acc.check_finite(got[b, :nv])
            for r0, r1 in voc_ref.windows(nv, tile):
                y64, m = voc_ref.conv_ref(xs_i[b], ws[i], bs[i], rs_i[b] if use_res else None, None, nv, r0, r1, dils[i])
                acc.add(got[b, r0:r1], y64, m)
    row.update(acc.row(), pad_untouched=pad, bitwise_vs_own_launches=eq)
    if use_res and n == 3 and mode != 2:
        # the grouped last layer of a stage (members in place into their own tensors) + gp_sum_div == three accumulating launches
        full = torch.empty(B, C // 4, L, 4, device=dev)
        rc_s = lib.ev_op_gp_sum_div(R.ptr(grp[0]), R.ptr(grp[1]), R.ptr(grp[2]), R.ptr(full), B * L * C, 3.0, R.st)
        accd = torch.full_like(full, float("nan"))
        res_d = [t.to(dev) for t in before]
        rca = [_conv_launch(R, mode, xg[i], wd[i], bd[i], res_d[i], accd, B, L, C, Ks[i], dils[i], lens_d, mul, acc=(0, 1, 2)[i], div=3.0)
               for i in range(n)]
        torch.cuda.synchronize()
        row["bitwise_sum_pass"] = rc_s == 0 and not any(rca) and _gp_valid_equal(full.cpu(), accd.cpu(), valid)
    return row


def run_pair_group(R, c, mode, seed):
    import torch
    import voc_plans as vp
    import voc_ref
    from emotivoice_b200 import layout
    lib, dev = R.lib, R.dev
    B, L, C, Ks, dils = c["B"], c["L"], c["C"], list(c["Ks"]), list(c["dils"])
    n = len(Ks)
    pl = vp.pair_group_plan(lib, Ks, dils, B, L, C, mode)
    solo_pl = [vp.pair_plan(lib, B, L, C, K, d, mode) for K, d in zip(Ks, dils)]
    row = dict(plan=pl and list(pl["key"]), L=L, member_mt=[p["MT"] if p else 0 for p in solo_pl])
    MT = pl["MT"] if pl else 2
    Rmin = 128 * MT - (max(Ks) - 1)
    mul = odd_mul(Rmin)
    # every member has its own rows per tile R = 128 MT - (K - 1): aim the lengths at the heaviest member's edges
    lens = pick_lens(B, L, Rmin, (0, 1, Rmin - 1), mul, tiny=(B >= 3)) if B > 1 else None
    if B == 1:
        k = (L - 1) // Rmin
        while k >= 0 and (k * Rmin + 1) % mul:
            k -= 1
        lens = [max(1, (k * Rmin + 1) // mul)]
    valid = [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    bf = mode == 2
    xs = [_nan_past(torch.randn(B, L, C, generator=g), valid) for _ in range(n)]
    w1s = [torch.randn(K, C, C, generator=g) / math.sqrt(C * K) for K in Ks]
    w2s = [torch.randn(K, C, C, generator=g) / math.sqrt(C * K) for K in Ks]
    b1s = [torch.randn(C, generator=g) for _ in range(n)]
    b2s = [torch.randn(C, generator=g) for _ in range(n)]
    pk = _pack(mode)
    w1d, w2d = [pk(w).to(dev) for w in w1s], [pk(w).to(dev) for w in w2s]
    b1d, b2d = [t.to(dev) for t in b1s], [t.to(dev) for t in b2s]
    xg = [layout.to_gp(x, bf).to(dev) for x in xs]
    before = layout.to_gp(torch.full((B, L, C), float("nan")), bf)
    grp = [before.to(dev) for _ in range(n)]
    solo = [before.to(dev) for _ in range(n)]
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    rcs = [lib.ev_op_resblock_gp(R.ptr(xg[i]), R.ptr(w1d[i]), R.ptr(b1d[i]), R.ptr(w2d[i]), R.ptr(b2d[i]), mode, R.ptr(solo[i]), B, L, C, Ks[i], dils[i],
                                 R.ptr(lens_d), mul, 0, 1.0, R.st) for i in range(n)]
    IA = ctypes.c_int * n
    rc = lib.ev_op_resblock_gp_group(n, _tab(R, xg), _tab(R, w1d), _tab(R, b1d), _tab(R, w2d), _tab(R, b2d), mode, _tab(R, grp), B, L, C, IA(*Ks), IA(*dils),
                                     R.ptr(lens_d), mul, R.st)
    torch.cuda.synchronize()
    row.update(rc=rc, solo_rc=rcs, lens=lens, lens_mul=mul)
    if pl is None:
        # a member whose own plan keeps fewer than two accumulators per tile is never grouped: the launch must refuse
        return dict(row, unsupported=True)
    if rc != 0 or any(rcs):
        return dict(row, err=R.err())
    acc = Acc(mode)
    eq, pad = True, True
    rnd = (lambda t: t.float().to(torch.bfloat16).double()) if bf else None
    for i in range(n):
        got_gp = grp[i].cpu()
        got = layout.from_gp(got_gp)
        pad = pad and _pad_ok(got_gp, before, valid)
        eq = eq and _gp_valid_equal(got_gp, solo[i].cpu(), valid)
        xs_i = _stored(xs[i], bf)
        Ri = 128 * MT - (Ks[i] - 1)
        for b, nv in enumerate(valid):
            acc.check_finite(got[b, :nv])
            for r0, r1 in voc_ref.windows(nv, Ri):
                y64, m = voc_ref.pair_ref(xs_i[b], w1s[i], b1s[i], w2s[i], b2s[i], None, nv, r0, r1, dils[i], 0, 1.0, xt_round=rnd)
                acc.add(got[b, r0:r1], y64, m)
    row.update(acc.row(), pad_untouched=pad, bitwise_vs_own_launches=eq)
    if n == 3 and mode != 2:
        full = torch.empty(B, C // 4, L, 4, device=dev)
        rc_s = lib.ev_op_gp_sum_div(R.ptr(grp[0]), R.ptr(grp[1]), R.ptr(grp[2]), R.ptr(full), B * L * C, 3.0, R.st)
        accd = before.to(dev)
        rca = [lib.ev_op_resblock_gp(R.ptr(xg[i]), R.ptr(w1d[i]), R.ptr(b1d[i]), R.ptr(w2d[i]), R.ptr(b2d[i]), mode, R.ptr(accd), B, L, C, Ks[i], dils[i],
                                     R.ptr(lens_d), mul, (0, 1, 2)[i], 3.0, R.st) for i in range(n)]
        torch.cuda.synchronize()
        row["bitwise_sum_pass"] = rc_s == 0 and not any(rca) and _gp_valid_equal(full.cpu(), accd.cpu(), valid)
    return row


TAU_POST = 2.0 ** -14        # conv_post: an fp32 FMA chain of K*C = 224 terms, ~2^-16 of the magnitude, on the values the kernel reads
TANH_ABS = 2.0 ** -20        # tanhf: a few ulps of a result <= 1


def run_post(R, c, seed):
    import torch
    import voc_ref
    from emotivoice_b200 import layout
    lib, dev = R.lib, R.dev
    B, L, C, K, mul, bf = c["B"], c["L"], c["C"], c["K"], c["mul"], c["bf"]
    lens = c["lens"]
    valid = [L] * B if lens is None else [min(L, v * mul) for v in lens]
    g = torch.Generator().manual_seed(seed)
    x = _nan_past(torch.randn(B, L, C, generator=g) * 2, valid)
    w = torch.randn(K, C, generator=g) * 0.1
    bias = torch.randn(1, generator=g)
    xg, wd, bd = layout.to_gp(x, bool(bf)).to(dev), w.to(dev), bias.to(dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev) if lens is not None else None
    wav = torch.full((B, L), float("nan"), device=dev)
    rc = lib.ev_op_conv_post_gp(R.ptr(xg), bf, R.ptr(wd), R.ptr(bd), R.ptr(lens_d), mul, B, L, C, K, 0.01, R.ptr(wav), R.st)
    torch.cuda.synchronize()
    row = dict(rc=rc, lens=lens, L=L)
    if rc != 0:
        return dict(row, err=R.err())
    got = wav.cpu()
    xs = _stored(x, bool(bf))
    err_m, fin, zero = 0.0, True, True
    for b, n in enumerate(valid):
        y64, m = voc_ref.post_ref(xs[b], w, bias, n)
        fin = fin and bool(torch.isfinite(got[b, :n]).all())
        e = ((got[b, :n].double() - y64).abs() - TANH_ABS) / m
        err_m = max(err_m, float(e.max()) if fin else float("inf"))
        zero = zero and bool((got[b, n:] == 0).all())
    return dict(row, err_m=err_m, finite=fin, pad_zero=zero, bound_ok=bool(fin and err_m <= TAU_POST))


def run_to_gp(R, bf, seed):
    import torch
    from emotivoice_b200 import layout
    g = torch.Generator().manual_seed(seed)
    mel = torch.randn(2, 80, 37, generator=g)
    mel_d = mel.to(R.dev)
    cpg = 8 if bf else 4
    outg = torch.empty((2, 80 // cpg, 37, cpg), dtype=torch.bfloat16 if bf else torch.float32, device=R.dev)
    rc = R.lib.ev_op_to_gp(R.ptr(mel_d), 80 * 37, 1, 37, R.ptr(outg), 2, 37, 80, bf, R.st)
    torch.cuda.synchronize()
    eq = rc == 0 and _bits(outg.cpu()).equal(_bits(layout.to_gp(mel.transpose(1, 2).contiguous(), bool(bf))))
    return dict(rc=rc, bitwise_vs_host=eq)


def main(family):
    lib = _setup()
    import torch
    R = Runner(lib)
    runner = {"conv": run_conv, "pair": run_pair, "group": run_group, "pair_group": run_pair_group}.get(family)
    if family == "post":
        for i, (cid, c) in enumerate(zip(case_ids("post"), _post_cases())):
            print(json.dumps(dict(id=cid, **run_post(R, c, 100 + i))), flush=True)
        for bf in (0, 1):
            print(json.dumps(dict(id="post-to_gp-bf%d" % bf, **run_to_gp(R, bf, 5 + bf))), flush=True)
        return
    for i, c in enumerate(FAMILIES[family]()):
        for mode in MODES:
            cid = "%s-%s-m%d" % (family, c["name"], mode)
            try:
                row = runner(R, c, mode, 1000 * i + 17 * mode + 1)
            except Exception as e:      # a Python-side error in one case must not hide the others' rows
                row = dict(exception="%s: %s" % (type(e).__name__, e))
            print(json.dumps(dict(id=cid, mode=mode, **row)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main(sys.argv[1])
