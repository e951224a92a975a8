"""Times the watermark on the GPU and measures how strongly it is detected.

- Embed: JETSGenerator.format_audio with and without ``watermark=`` (one ev_watermark_embed launch ahead of the chain), on the
  b1_t100 fixture's utterance at B=1 and a cfg3-like batch (B=32, 20..200 phonemes), each at 24 kHz pcm16 and 8 kHz mu-law.
  CUDA events around --iters calls after --warmup, mean per call on the device timeline; the variants alternate (plain,
  marked, plain again: the two plain runs give the spread).
- Detect: watermark.detect on 3 s, 10 s and 60 s recordings and on 32 x 10 s, at 16 kHz, timed the same way.
- z against clip length: seeded speech-like signals (tests/test_watermark.py) marked through format_audio in each output
  format, plain and with loudness -16 / true peak -1, decoded, cut to each length from the start and detected; the smallest z
  over five signals per length.  Also the largest peak increase the mark causes without true_peak (16 kHz float32).

    python tools/watermark_timing.py [--iters 100] [--warmup 10] [--out profiles/h100_watermark_timing.json]

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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from emotivoice_b200 import frontdoor as fd                 # noqa: E402
from emotivoice_b200 import synth, watermark                # noqa: E402
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402
from test_watermark import speech_like                      # noqa: E402
from test_watermark_gpu import FORMATS, _decode             # noqa: E402

KEY = 0x5EEDCAFEF00D
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
LENGTHS_S = (2.0, 3.0, 4.0, 5.0, 6.0, 8.0, 10.0, 12.0, 15.0)


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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_watermark_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the watermark kernels run on the GPU only")
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
    embed = {}
    for name, batch in workloads.items():
        out = model(**batch)
        torch.cuda.synchronize()
        n_in = [int(n) * 256 for n in out["mel_lengths_host"].tolist()]
        embed[name] = {"batch": len(n_in), "samples_in": sum(n_in)}
        for rate, enc in ((24000, "pcm16"), (8000, "mulaw")):
            p1 = device_ms(lambda: model.format_audio(out, rate, enc), args.iters, args.warmup)
            m = device_ms(lambda: model.format_audio(out, rate, enc, watermark=KEY), args.iters, args.warmup)
            p2 = device_ms(lambda: model.format_audio(out, rate, enc), args.iters, args.warmup)
            r = {"gpu_ms_per_call_plain": round(min(p1, p2), 4), "gpu_ms_per_call_marked": round(m, 4),
                 "watermark_extra_ms": round(m - min(p1, p2), 4), "plain_repeat_spread_ms": round(abs(p1 - p2), 4)}
            embed[name]["%d_%s" % (rate, enc)] = r
            print("embed", name, rate, enc, json.dumps(r), flush=True)
    detect = {}
    for name, (B, secs) in {"3s": (1, 3), "10s": (1, 10), "60s": (1, 60), "32x10s": (32, 10)}.items():
        w = torch.from_numpy(np.random.default_rng(4).standard_normal((B, secs * 16000)).astype(np.float32) * 0.1).to(dev)
        ms = device_ms(lambda: watermark.detect(w, 16000, KEY), max(3, args.iters // 10), 2)
        detect[name] = round(ms, 3)
        print("detect", name, ms, flush=True)
    sigs = [speech_like(max(LENGTHS_S), 700 + i) for i in range(5)]
    w = np.stack(sigs)[:, None, :]
    out = {"wav_predictions": torch.from_numpy(w).to(dev), "mel_lengths_host": torch.tensor([w.shape[-1]] * len(sigs))}
    ztab = {}
    for rate, enc in FORMATS:
        for chain_name, chain in (("plain", {}), ("loud-16_tp-1", dict(loudness=-16.0, true_peak=-1.0))):
            marked = [_decode(x, rate, enc) for x in fd.fetch_audio(model, out, rate, enc, hop=1, **chain, watermark=KEY)]
            row = {}
            for s in LENGTHS_S:
                n = int(round(s * rate))
                xs = np.stack([m[:n] for m in marked]).astype(np.float32)
                z = watermark.detect(torch.from_numpy(xs).to(dev), rate, KEY)[0].cpu().numpy()
                row["%gs" % s] = [round(float(z.min()), 2), round(float(z.mean()), 2)]
            ztab["%d_%s_%s" % (rate, enc, chain_name)] = row
            print("z", rate, enc, chain_name, json.dumps(row), flush=True)
    plain = fd.fetch_audio(model, out, 16000, "float32", hop=1)
    marked = fd.fetch_audio(model, out, 16000, "float32", hop=1, watermark=KEY)
    peak_db = max(20 * np.log10(np.max(np.abs(m)) / np.max(np.abs(p))) for p, m in zip(plain, marked))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), key=KEY, iters=args.iters, warmup=args.warmup, embed=embed, detect_ms=detect,
               z_min_mean_by_length=ztab, largest_peak_increase_db=round(float(peak_db), 3))
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
