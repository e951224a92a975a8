"""A/B timing of the acoustic model's GEMM-shaped launches (conv1d_tc, with its split-K reduce) between two builds of the engine,
in one process, alternating the builds launch by launch.

    python tools/ab_am.py [--a LIB.so | --base REV] [--b LIB.so] [--rounds 20] [--phonemes 100] [--frames 512]
                          [--precisions fp32,tf32,bf16] [--out DIR]

A is `--a`, or else revision REV (default HEAD~1) exported with `git archive` and built in a temporary directory; B is `--b`, or else
the in-tree library (built if stale).  Both libraries are loaded side by side.  The layers are those of bench.py's headline step at
batch 1 (T phonemes, F mel frames): the encoder, the conditioning and the predictors (3xTF32 in every precision), the decoder and
to_mel (bf16x3 in "fp32", 1xTF32 in "tf32", bf16 in "bf16"), each with the engine's K-split factor, bias, activation and in-place
residual (tests/am_plans.py restates the engine's launch list).  The engine's own planner picks every tile.  Per precision, round
and layer, each build runs the same launch on its own copy of the same seeded inputs, with the L2 flushed before every launch and
CUDA events around it; the build that goes first alternates between rounds.  Prints the card's name, power limit and max SM clock
(read in the same run) and, per layer, the plan, both builds' median times and B's median over A's, then the per-step sum (each
layer's median times the launches of it in one step).  With --out DIR the times go to DIR/ab_am.json.
"""
import argparse
import json
import math
import os
import statistics
import sys
import tempfile
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def layer_launches(B, T, F, prec):
    """name -> (layer record of am_plans.am_layers, launches per step) for the distinct convolutions of one step"""
    import am_plans
    out = OrderedDict()
    for r in am_plans.am_layers(B, T, F, prec, invariant=False):
        if isinstance(r, dict):
            if r["name"] in out:
                out[r["name"]][1] += 1
            else:
                out[r["name"]] = [r, 1]
    return out


def make_launch(lib, dev, r, seed):
    """The launch of one layer record on seeded inputs: returns a closure that issues it (the convolution and, when the plan splits
    K, its reduce) on the current stream"""
    from emotivoice_b200 import packing
    import am_plans
    B, L, Cin, Cout, K, mode, S = r["B"], r["L"], r["Cin"], r["Cout"], r["K"], r["mode"], r["ksplit"]
    pl = am_plans.tc_plan(lib, B, L, Cin, Cout, K, mode, S)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, Cin, generator=g).to(dev)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    pack = packing.to_tc16x2_layout if mode == 3 else (packing.to_tc16_layout if mode == 2 else packing.to_tc_layout)
    wd = pack(w).to(dev)
    bias = torch.randn(B if r["bias_bs"] else 1, Cout, generator=g).to(dev)
    out = torch.randn(B, L, Cout, generator=g).to(dev)          # also the residual of the in-place layers, as in the engine
    ws = torch.empty(pl["S"] * B * L * Cout, device=dev) if pl["S"] > 1 else None
    st = torch.cuda.current_stream().cuda_stream
    res = out.data_ptr() if r["inplace"] else None
    keep = (x, wd, bias, out, ws)

    def call():
        return lib.ev_op_conv1d_tc_ks(x.data_ptr(), wd.data_ptr(), mode, bias.data_ptr(), r["bias_bs"], res, out.data_ptr(), B, L, Cin,
                                      Cout, K, 1, None, 1, 0, 0.0, r["out_act"], 0, 1.0, S, None if ws is None else ws.data_ptr(),
                                      0 if ws is None else ws.numel(), st)
    return dict(call=call, keep=keep, plan=pl, flops=2.0 * B * L * Cin * Cout * K)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", default=None, help="library A (default: --base built from git)")
    ap.add_argument("--base", default="HEAD~1", help="revision built as A when --a is not given")
    ap.add_argument("--b", default=None, help="library B (default: the in-tree library)")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--phonemes", type=int, default=100)
    ap.add_argument("--frames", type=int, default=512, help="mel frames of the utterance; bench.py's step has about 512")
    ap.add_argument("--precisions", default="fp32,tf32,bf16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ab_am.py needs a CUDA device"

    from ab_dominant import build_revision, load
    from profile_step import card
    from emotivoice_b200 import _abi, build

    with tempfile.TemporaryDirectory() as keep_dir:
        path_a = args.a or build_revision(args.base, keep_dir)
        path_b = args.b or build.build(verbose=False)
        libs = {"A": load(path_a), "B": load(path_b)}
        dev = torch.device("cuda", 0)
        flush_buf = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
        info = card()
        print("%s, power limit %s, max SM clock %s" % (info["name"], info["power_limit"], info["sm_max_clock"]))
        print("A = %s\nB = %s" % (path_a if args.a else "%s (%s)" % (args.base, path_a), path_b))
        print("batch 1, %d phonemes, %d mel frames; %d rounds, L2 flushed before every launch" % (args.phonemes, args.frames, args.rounds))
        res = {"card": info, "a": path_a, "b": path_b, "phonemes": args.phonemes, "frames": args.frames, "precisions": {}}

        def once(d):
            flush_buf.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _abi.check(d["call"]())
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) * 1e3          # us

        for prec in args.precisions.split(","):
            layers = layer_launches(1, args.phonemes, args.frames, prec)
            runs = {name: {k: make_launch(lib, dev, r, 1000 + i) for k, lib in libs.items()} for i, (name, (r, _)) in enumerate(layers.items())}
            for name in layers:
                for _ in range(args.warmup):
                    once(runs[name]["A"]), once(runs[name]["B"])
            ts = {name: {"A": [], "B": []} for name in layers}
            for rnd in range(args.rounds):
                for name in layers:
                    for k in (("A", "B") if rnd % 2 == 0 else ("B", "A")):
                        ts[name][k].append(once(runs[name][k]))
            print("%s:" % prec)
            print("  %-12s %4s  %-34s %9s %9s %7s" % ("layer", "n", "plan (MODE, MT, KBG, BN, A, B, groups, S)", "A us", "B us", "B/A"))
            tot = {"A": 0.0, "B": 0.0}
            rows = OrderedDict()
            for name, (r, n) in layers.items():
                med = {k: statistics.median(v) for k, v in ts[name].items()}
                for k in tot:
                    tot[k] += n * med[k]
                key = runs[name]["B"]["plan"]["key"]
                print("  %-12s %4d  %-34s %9.1f %9.1f %7.3f" % (name, n, str(tuple(key)), med["A"], med["B"], med["B"] / med["A"]))
                rows[name] = {"launches_per_step": n, "plan": list(key), "flops": runs[name]["B"]["flops"], "us": ts[name],
                              "median_ratio_b_over_a": med["B"] / med["A"]}
            print("  per step (sum of median x launches): A %.1f us, B %.1f us, B/A %.3f" % (tot["A"], tot["B"], tot["B"] / tot["A"]))
            res["precisions"][prec] = {"layers": rows, "per_step_us": tot}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_am.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
