"""Where the device time of the headline step goes: bench.py's workload (B=1, 100-phoneme corpus utterances, fp32 mode by default,
L2 flushed between steps) under torch.profiler with CUDA activities, in a run of its own.

    python tools/profile_step.py [--steps 20] [--warmup 5] [--precision fp32] [--out DIR]

Prints, per step: device time of every kernel (name with template arguments), its launches and its share of the summed kernel time,
then the total of each stage.  The three engine calls (`ev:am_phase1`, `ev:am_phase2`, `ev:vocoder`, the engine's NVTX range names)
are wrapped in profiler ranges on the host, and a kernel belongs to the range its launch was issued in.  The vocoder's stages
(`voc:stage1..4`) are NVTX ranges inside one engine call; torch.profiler does not record NVTX ranges, so they are not split out here.
With programmatic dependent launch (the default) a kernel's span starts while its predecessor still runs and includes its wait for
it, so spans overlap and their sum exceeds the step time; run with EV_PDL=0 for spans that do not overlap.
The card's name and power limit are read in the same run.  With --out DIR the table is also written as DIR/profile_step.json; the
raw trace goes to a temporary directory and is deleted.
"""
import argparse
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

PHASES = (("ev_am_phase1", "ev:am_phase1"), ("ev_am_phase1_prosody", "ev:am_phase1"), ("ev_am_phase2", "ev:am_phase2"),
          ("ev_vocoder", "ev:vocoder"))
N_PHONEMES = 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, sm_max_clock=clk)
    except Exception as e:
        return dict(name=torch.cuda.get_device_name(), power_limit="unknown (%s)" % repr(e)[:80], sm_max_clock="unknown")


def short_name(n):
    n = re.sub(r"^void ", "", n)
    depth, out = 0, []
    for ch in n:          # drop the parameter list, keep the template arguments
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            break
        out.append(ch)
    return "".join(out).strip()


def wrap_phases(lib):
    """Every engine call runs inside a profiler range named after the NVTX range the engine opens in it."""
    for sym, rng in PHASES:
        fn = getattr(lib, sym)

        def call(*a, _fn=fn, _rng=rng):
            with torch.profiler.record_function(_rng):
                return _fn(*a)
        setattr(lib, sym, call)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "tf32", "bf16", "fp32_ffma"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_step.py needs a CUDA device"

    import __graft_entry__  # noqa: F401
    from emotivoice_b200 import build as _build
    _build.build(verbose=False)
    from emotivoice_b200.config import default_config
    from emotivoice_b200 import synth, _abi
    from emotivoice_b200.modules import JETSGenerator

    dev = torch.device("cuda", 0)
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    model.precision = args.precision
    wrap_phases(_abi.load())
    model.reserve(batch=1, phonemes=N_PHONEMES + 28, frames=1024)
    n = args.warmup + args.steps
    batches = [{k: v.to(dev) for k, v in synth.collate_utterances([synth.corpus_utterance(i, n_phonemes=N_PHONEMES)]).items()}
               for i in range(n)]
    flush_buf = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    for s in range(args.warmup):
        model(**batches[s])
    torch.cuda.synchronize()

    frames = 0
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with tempfile.TemporaryDirectory() as tmp:
        with torch.profiler.profile(activities=acts) as prof:
            for s in range(args.steps):
                flush_buf.zero_()
                with torch.profiler.record_function("ev:step"):
                    out = model(**batches[args.warmup + s])
                frames += int(out["dec_outputs"].shape[1])
            torch.cuda.synchronize()
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    info = card()

    ranges = sorted([(e["ts"], e["ts"] + e["dur"], e["name"]) for e in ev if e.get("ph") == "X" and e.get("cat") == "user_annotation"
                     and e["name"] in ("ev:am_phase1", "ev:am_phase2", "ev:vocoder")])
    launch_at = {e["args"]["correlation"]: e["ts"] for e in ev if e.get("ph") == "X" and e.get("cat") == "cuda_runtime"
                 and "correlation" in e.get("args", {})}
    kernels = sorted([e for e in ev if e.get("ph") == "X" and e.get("cat") == "kernel"], key=lambda e: e["ts"])

    def phase_of(k):
        t = launch_at.get(k["args"].get("correlation"))
        if t is None:
            return None
        for a, b, name in ranges:
            if a <= t <= b:
                return name
        return None

    per_kernel = OrderedDict()
    phase_us = OrderedDict((p, 0.0) for p in ("ev:am_phase1", "ev:am_phase2", "ev:vocoder"))
    total = 0.0
    for k in kernels:
        ph = phase_of(k)
        if ph is None:
            continue                   # the L2 flush between steps and anything else outside the engine
        name = short_name(k["name"])
        a = per_kernel.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += k["dur"]
        phase_us[ph] += k["dur"]
        total += k["dur"]

    S = args.steps
    res = {"card": info, "precision": args.precision, "steps": S, "mel_frames_per_step": frames / S,
           "kernel_us_per_step": total / S, "launches_per_step": sum(v[0] for v in per_kernel.values()) / S,
           "kernels": [{"name": k, "us_per_step": v[1] / S, "share": v[1] / total, "launches_per_step": v[0] / S}
                       for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1][1])],
           "phases": [{"name": p, "us_per_step": v / S, "share": v / total} for p, v in phase_us.items()]}

    print("%s, power limit %s, max SM clock %s; precision %s, %d profiled steps, %.0f mel frames per step"
          % (info["name"], info["power_limit"], info["sm_max_clock"], args.precision, S, frames / S))
    print("kernel time %.1f us per step over %.1f launches (summed spans, which overlap under PDL; the L2 flush between steps excluded)"
          % (res["kernel_us_per_step"], res["launches_per_step"]))
    print("%7s  %10s  %9s  %s" % ("share", "us/step", "launches", "kernel"))
    for k in res["kernels"]:
        print("%6.1f%%  %10.1f  %9.1f  %s" % (100 * k["share"], k["us_per_step"], k["launches_per_step"], k["name"]))
    print("stage totals:")
    for p in res["phases"]:
        print("%6.1f%%  %10.1f  %s" % (100 * p["share"], p["us_per_step"], p["name"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "profile_step.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
