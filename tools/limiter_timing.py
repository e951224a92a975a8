"""Times the true-peak limiter on the GPU: JETSGenerator.format_audio with ``loudness=-16`` against ``loudness=-16,
true_peak=-1`` (two ev_loudness measurements and two ev_limit passes ahead of the format launch, instead of one measurement).

Workloads as tools/loudness_timing.py: the b1_t100 fixture's utterance at B=1, and a cfg3-like batch (B=32, 20..200 phonemes),
each at 8 kHz mu-law and 24 kHz pcm16.  CUDA events around --iters format_audio calls after --warmup, mean per call on the
device timeline; the two variants alternate per workload and format.

    python tools/limiter_timing.py [--iters 200] [--warmup 20] [--out profiles/h100_limiter_timing.json]

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

from emotivoice_b200 import synth                           # noqa: E402
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402

FORMATS = [(8000, "mulaw"), (24000, "pcm16")]
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
TARGET, CEILING = -16.0, -1.0


def device_ms(fn, iters, warmup):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_limiter_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the limiter kernels run on the GPU only")
    dev = torch.device("cuda:0")
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    g = np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz"))
    b1 = {k: torch.from_numpy(g[k]).to(dev) for k in KEYS}
    rng = np.random.default_rng(32)
    lens = sorted(rng.integers(20, 201, size=32).tolist(), reverse=True)
    workloads = {"b1_fixture": b1, "cfg3_b32": {k: v.to(dev) for k, v in synth.make_batch(lens, seed=3232).items()}}
    res = {}
    for name, batch in workloads.items():
        out = model(**batch)
        torch.cuda.synchronize()
        n_in = [int(n) * 256 for n in out["mel_lengths_host"].tolist()]
        res[name] = {"batch": len(n_in), "samples_in": sum(n_in)}
        for rate, enc in FORMATS:
            loud_ms = device_ms(lambda: model.format_audio(out, rate, enc, loudness=TARGET), args.iters, args.warmup)
            lim_ms = device_ms(lambda: model.format_audio(out, rate, enc, loudness=TARGET, true_peak=CEILING), args.iters, args.warmup)
            loud_ms2 = device_ms(lambda: model.format_audio(out, rate, enc, loudness=TARGET), args.iters, args.warmup)
            r = {"gpu_ms_per_call_loudness": round(min(loud_ms, loud_ms2), 4), "gpu_ms_per_call_loudness_true_peak": round(lim_ms, 4),
                 "true_peak_extra_ms": round(lim_ms - min(loud_ms, loud_ms2), 4),
                 "loudness_repeat_spread_ms": round(abs(loud_ms - loud_ms2), 4)}
            res[name]["%d_%s" % (rate, enc)] = r
            print(name, rate, enc, json.dumps(r), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), target_lufs=TARGET, true_peak_dbtp=CEILING, iters=args.iters, warmup=args.warmup, results=res)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
