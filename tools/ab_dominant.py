"""A/B timing of bench.py's dominant launch (bench.dominant_launch: the grouped stage-2 ResBlock convolutions of the batch-1 step)
between two builds of the engine, in one process, alternating the builds launch by launch.

    python tools/ab_dominant.py [--a LIB.so | --base REV] [--b LIB.so] [--rounds 20] [--frames 511] [--precisions fp32,tf32,bf16]
                                [--out DIR]

A is `--a`, or else revision REV (default HEAD~1) exported with `git archive` and built in a temporary directory; B is `--b`, or else
the in-tree library (built if stale).  Both libraries are loaded side by side.  Per precision and round, each build runs the same
launch on its own copy of the same seeded inputs, with the L2 flushed before every launch and CUDA events around it; the build
that goes first alternates between rounds.  Prints the card's name, power limit and max SM clock (read in the same run) and, per
precision, both builds' times (min / median / max) and B's median over A's.  With --out DIR the times go to DIR/ab_dominant.json.
"""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402


def build_revision(rev, dst_dir):
    """`git archive rev` -> a temporary tree -> its own build; returns the library copied to dst_dir"""
    with tempfile.TemporaryDirectory() as tmp:
        archive = subprocess.run(["git", "-C", ROOT, "archive", rev], capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=archive, check=True)
        subprocess.run([sys.executable, "-m", "emotivoice_b200.build"], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
        out = os.path.join(dst_dir, "lib_%s.so" % rev.replace("/", "_").replace("~", "_"))
        shutil.copy(os.path.join(tmp, "emotivoice_b200", "lib", "libemotivoice_b200.so"), out)
        return out


def load(path):
    from emotivoice_b200 import _abi
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _abi.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", default=None, help="library A (default: --base built from git)")
    ap.add_argument("--base", default="HEAD~1", help="revision built as A when --a is not given")
    ap.add_argument("--b", default=None, help="library B (default: the in-tree library)")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=511, help="mel frames of the utterance (L = 64 frames); bench.py's step has ~511")
    ap.add_argument("--precisions", default="fp32,tf32,bf16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ab_dominant.py needs a CUDA device"

    import bench
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
        res = {"card": info, "a": path_a, "b": path_b, "frames": args.frames, "precisions": {}}
        for prec in args.precisions.split(","):
            d = {k: bench.dominant_launch(lib, dev, args.frames, prec) for k, lib in libs.items()}

            def once(k):
                flush_buf.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _abi.check(d[k]["call"]())
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
            print("%s: %s" % (prec, d["A"]["kname"]))
            for k in ("A", "B"):
                v = sorted(ts[k])
                print("  %s: min %.1f  median %.1f  max %.1f us  (%d launches; %.1f algorithmic TFLOP/s at the median)"
                      % (k, v[0], med[k], v[-1], len(v), d[k]["flops"] / med[k] / 1e6))
            print("  B / A median: %.3f" % (med["B"] / med["A"]))
            res["precisions"][prec] = {"kernel": d["A"]["kname"], "flops": d["A"]["flops"], "us": ts, "median_ratio_b_over_a": med["B"] / med["A"]}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_dominant.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
