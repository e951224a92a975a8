"""Times feats.Pitch.get_pitch (one ev_pitch call: DIO, StoneMask and the continuous interpolation, fp64) at the config
(16 kHz, hop 256) on the GPU, beside the fp64 numpy restatement of pyworld.dio + pyworld.stonemask (oracle/pitch_oracle.py) on the
host CPU.  The CPU figure is the restatement's, not pyworld's: pyworld is not installed and was never timed.

Workloads: B=1 on the b1_t100 fixture's 8.6 s waveform; B=32 seeded voiced items of 1-10 s (harmonic complexes with vibrato
over a -80 dBFS floor), padded to the longest with per-item lengths.  GPU: CUDA events around --iters calls after --warmup, mean
per call on the device timeline, the whole get_pitch chain (dtype cast, workspace, launches).  CPU: the mean of --cpu-iters
runs of the restatement, per item, summed over the batch.

    python tools/pitch_timing.py [--iters 200] [--warmup 20] [--cpu-iters 1] [--out FILE]

Prints one JSON line with the GPU name and power limit (read in the same run); --out also writes it to FILE."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200 import feats                           # noqa: E402
from oracle import pitch_oracle as PO                       # noqa: E402

SR, HOP = 16000, 256


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def voiced(n, rng):
    t = np.arange(n) / SR
    f0 = rng.uniform(90, 300)
    ph = 2 * np.pi * np.cumsum(f0 * (1 + 0.04 * np.sin(2 * np.pi * 5 * t))) / SR
    return (sum(0.3 / k * np.sin(k * ph) for k in range(1, 6)) + 1e-4 * rng.standard_normal(n)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--cpu-iters", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: ev_pitch runs on the GPU only")
    dev = torch.device("cuda:0")
    with np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz")) as z:
        b1 = z["wav"].reshape(-1).astype(np.float32)
    rng = np.random.default_rng(3233)
    lens = rng.integers(1 * SR, 10 * SR + 1, size=32).tolist()
    items = [voiced(n, rng) for n in lens]
    workloads = {"b1_fixture": ([b1], None), "b32_1to10s": (items, lens)}
    P = feats.Pitch(sr=SR, hop_length=HOP)
    res = {}
    for name, (its, ls) in workloads.items():
        N = max(len(x) for x in its)
        y = torch.zeros(len(its), N)
        for b, x in enumerate(its):
            y[b, :len(x)] = torch.from_numpy(x)
        y = y.to(dev)
        ms = timed(lambda: P.get_pitch(y, lengths=ls), args.iters, args.warmup)
        out = P.get_pitch(y, lengths=ls).cpu().numpy()
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            want = [PO.continuous(PO.pitch(x.astype(np.float64), SR, HOP)[1]) for x in its]
        cpu_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        rel = max(float(np.max(np.abs(out[b, :len(w)] - w) / np.maximum(np.abs(w), 1e-300))) for b, w in enumerate(want))
        voiced_frames = int(sum((o != 0).sum() for o in out))
        res[name] = {"batch": len(its), "samples": sum(len(x) for x in its), "frames": sum(len(x) // HOP + 1 for x in its),
                     "nonzero_frames": voiced_frames, "get_pitch_gpu_ms": round(ms, 4),
                     "restatement_numpy_cpu_ms": round(cpu_ms, 1), "max_rel_diff_vs_restatement": rel}
        print(name, json.dumps(res[name]), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    line = json.dumps(dict(gpu=q.stdout.strip(), cpu=os.cpu_count(), iters=args.iters, warmup=args.warmup, cpu_iters=args.cpu_iters,
                           results=res))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
