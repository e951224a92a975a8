"""A/B timing of the fused ResBlock layers of vocoder stages 3 and 4 (resblock_gp_kernel, C = 64 and C = 32) between two builds of the
engine, in one process, alternating the builds launch by launch.

    python tools/ab_resblock.py [--a LIB.so | --base REV] [--b LIB.so] [--rounds 20] [--frames 512] [--precisions fp32,tf32,bf16]
                                [--out DIR]

The launches are the engine's at batch 1: per stage and dilation index (1, 3, 5), ONE grouped launch of the same-index layers of
HiFi-GAN's three parallel ResBlocks (k = 11 / 7 / 3), stage 3 at C = 64, L = 128 F and stage 4 at C = 32, L = 256 F (F mel frames).
A is `--a`, or else revision REV (default HEAD~1) exported with `git archive` and built in a temporary directory; B is `--b`, or else
the in-tree library (built if stale).  Both libraries are loaded side by side.  Per precision, stage and round, each build runs the
stage's three grouped launches on its own copy of the same seeded inputs, with the L2 flushed before them and CUDA events around
them; the build that goes first alternates between rounds.  Prints the card's name, power limit and max SM clock (read in the same
run) and, per precision and stage, both builds' times (min / median / max) and B's median over A's.  With --out DIR the times go to
DIR/ab_resblock.json.
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

KS, DILS = (11, 7, 3), (1, 3, 5)
STAGES = (("stage3", 64, 128), ("stage4", 32, 256))      # name, channels, samples per mel frame


def stage_launches(lib, dev, C, L, precision):
    """the stage's three grouped fused launches (dilation index 1, 3, 5) as one closure, with its algorithmic FLOPs"""
    from emotivoice_b200 import _abi, layout, packing
    mode = {"fp32": 3, "tf32": 0, "bf16": 2}[precision]
    bf = mode == 2
    pack = packing.to_tc16x2_layout if mode == 3 else (packing.to_tc16_layout if bf else packing.to_tc_layout)
    g = torch.Generator().manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream
    n = len(KS)
    VP, IA = ctypes.c_void_p * n, ctypes.c_int * n
    keep, calls = [], []
    for d in DILS:
        w1 = [pack(torch.randn(K, C, C, generator=g) / math.sqrt(C * K)).to(dev) for K in KS]
        w2 = [pack(torch.randn(K, C, C, generator=g) / math.sqrt(C * K)).to(dev) for K in KS]
        b1 = [torch.randn(C, generator=g).to(dev) for _ in KS]
        b2 = [torch.randn(C, generator=g).to(dev) for _ in KS]
        x = [layout.to_gp(torch.randn(1, L, C, generator=g), bf).to(dev) for _ in KS]
        out = [torch.empty_like(t) for t in x]
        tabs = [VP(*[t.data_ptr() for t in ts]) for ts in (x, w1, b1, w2, b2, out)]
        keep += [w1, w2, b1, b2, x, out, tabs]
        calls.append(lambda tabs=tabs, d=d: lib.ev_op_resblock_gp_group(n, tabs[0], tabs[1], tabs[2], tabs[3], tabs[4], mode, tabs[5], 1, L, C,
                                                                        IA(*KS), IA(*([d] * n)), None, 1, st))

    def call():
        for c in calls:
            _abi.check(c())
    return dict(call=call, keep=keep, flops=len(DILS) * 2 * 2.0 * L * C * C * sum(KS))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", default=None, help="library A (default: --base built from git)")
    ap.add_argument("--base", default="HEAD~1", help="revision built as A when --a is not given")
    ap.add_argument("--b", default=None, help="library B (default: the in-tree library)")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=512, help="mel frames of the utterance; bench.py's step has ~511")
    ap.add_argument("--precisions", default="fp32,tf32,bf16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ab_resblock.py needs a CUDA device"

    from ab_dominant import build_revision, load
    from profile_step import card
    from emotivoice_b200 import build

    with tempfile.TemporaryDirectory() as keep_dir:
        path_a = args.a or build_revision(args.base, keep_dir)
        path_b = args.b or build.build(verbose=False)
        libs = {"A": load(path_a), "B": load(path_b)}
        dev = torch.device("cuda", 0)
        flush_buf = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
        info = card()
        print("%s, power limit %s, max SM clock %s" % (info["name"], info["power_limit"], info["sm_max_clock"]))
        print("A = %s\nB = %s" % (path_a if args.a else "%s (%s)" % (args.base, path_a), path_b))
        res = {"card": info, "a": path_a, "b": path_b, "frames": args.frames, "precisions": {}}
        for prec in args.precisions.split(","):
            res["precisions"][prec] = {}
            for stage, C, per_frame in STAGES:
                L = per_frame * args.frames
                d = {k: stage_launches(lib, dev, C, L, prec) for k, lib in libs.items()}

                def once(k):
                    flush_buf.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    d[k]["call"]()
                    e1.record()
                    e1.synchronize()
                    return e0.elapsed_time(e1) * 1e3          # us

                for _ in range(args.warmup):
                    once("A"), once("B")
                ts = {"A": [], "B": []}
                for r in range(args.rounds):
                    for k in (("A", "B") if r % 2 == 0 else ("B", "A")):
                        ts[k].append(once(k))
                med = {k: statistics.median(v) for k, v in ts.items()}
                print("%s %s: C=%d L=%d, 3 grouped launches (k = %s, dilation %s)" % (prec, stage, C, L, KS, DILS))
                for k in ("A", "B"):
                    v = sorted(ts[k])
                    print("  %s: min %.1f  median %.1f  max %.1f us  (%d rounds; %.1f algorithmic TFLOP/s at the median)"
                          % (k, v[0], med[k], v[-1], len(v), d[k]["flops"] / med[k] / 1e6))
                print("  B / A median: %.3f" % (med["B"] / med["A"]))
                res["precisions"][prec][stage] = {"C": C, "L": L, "flops": d["A"]["flops"], "us": ts, "median_ratio_b_over_a": med["B"] / med["A"]}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_resblock.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
