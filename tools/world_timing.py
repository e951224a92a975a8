"""Times WORLD spectral envelopes and paper-style MCD on the GPU (``feats.spectral_envelope``: one ev_world_envelope launch;
``evaluate.compare(cepstrum=...)``).

Cases, at 16 kHz, 32 items of 10 s:
- envelope_hop256 / envelope_hop80: ``spectral_envelope`` with caller F0 at hop 256 (16 ms) and hop 80 (5 ms, pyworld's
  default frame period), the envelope kernel alone; and with f0=None, which adds ``pitch_track``.
- compare_mel / compare_world: ``compare`` of each item against a recording 8 % longer, in both cepstrum kinds.
CUDA events around --iters calls after --warmup, mean per call on the device timeline; the per-kernel device times of
envelope_hop80 come from torch.profiler in a run of their own.  No CPU comparison: pyworld and pysptk are not dependencies.

    python tools/world_timing.py [--iters 10] [--warmup 2] [--out profiles/h100_world_timing.json]

Reads the GPU name and power limit in the same run; prints the record and writes it to --out."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200 import evaluate, feats                 # noqa: E402
from tools.evaluate_timing import device_ms, voiced          # noqa: E402

SR = 16000
B, SECONDS = 32, 10.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_world_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the envelope kernels run on the GPU only")
    dev = torch.device("cuda:0")
    syn = torch.from_numpy(np.stack([voiced(SECONDS, 2 * b) for b in range(B)])).to(dev)
    ref = torch.from_numpy(np.stack([voiced(SECONDS * 1.08, 2 * b + 1) for b in range(B)])).to(dev)
    rec = {"items": B, "samples": int(syn.shape[1]), "rate": SR}
    for hop in (256, 80):
        f0 = feats.pitch_track(syn, SR, hop, continuous=False)
        r = {"frames_per_item": int(f0.shape[1]), "fft_size": feats.world_fft_size(SR)}
        r["envelope_ms"] = round(device_ms(lambda: feats.spectral_envelope(syn, SR, hop, f0=f0), args.iters, args.warmup), 3)
        r["envelope_with_pitch_ms"] = round(device_ms(lambda: feats.spectral_envelope(syn, SR, hop), args.iters, args.warmup), 3)
        r["frames_per_ms"] = round(B * r["frames_per_item"] / r["envelope_ms"], 1)
        rec["envelope_hop%d" % hop] = r
        print("envelope_hop%d" % hop, json.dumps(r), flush=True)
        if hop == 80:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                feats.spectral_envelope(syn, SR, hop, f0=f0)
                torch.cuda.synchronize()
            r["kernel_ms"] = {e.key: round(e.device_time_total / 1000.0, 3) for e in prof.key_averages() if e.device_time_total > 0}
    for kind in ("mel", "world"):
        ms = device_ms(lambda: evaluate.compare(syn, ref, cepstrum=kind), args.iters, args.warmup)
        rec["compare_%s_ms" % kind] = round(ms, 3)
        print("compare_%s_ms" % kind, rec["compare_%s_ms" % kind], flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), iters=args.iters, warmup=args.warmup, cpu_comparison="not measured: pyworld and pysptk are "
               "not installed", **rec)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
