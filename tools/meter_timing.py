"""Times the loudness meter on the GPU (ev_meter: four launches).

Cases:
- b1_fixture: the b1_t100 fixture's output (137,472 samples, 8.6 s at 16 kHz), through ``loudness.meter`` on the waveform and
  through ``JETSGenerator.meter`` (the chain's float32 stage, one ev_format_audio launch, then ev_meter on its packed output),
  and ``JETSGenerator.format_audio(out, 16000, "float32")`` alone for comparison.
- b32_10s_16k: 32 recordings of 10 s of noise at 16 kHz, without and with the momentary / short-term series.
- one_hour_48k: one 60-minute recording at 48 kHz.
CUDA events around --iters calls after --warmup, mean per call on the device timeline (the lengths' H2D copy and the launches;
the samples are already on the device).

    python tools/meter_timing.py [--iters 100] [--warmup 10] [--out profiles/h100_meter_timing.json]

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

from emotivoice_b200 import loudness, synth                 # noqa: E402
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402

KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")


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
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_meter_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the meter kernels run on the GPU only")
    dev = torch.device("cuda:0")
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    g = np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz"))
    out = model(**{k: torch.from_numpy(g[k]).to(dev) for k in KEYS})
    torch.cuda.synchronize()
    n = int(out["mel_lengths_host"][0]) * 256
    wav = out["wav_predictions"][:, 0]
    it, wu = args.iters, args.warmup
    rec = {"b1_fixture": {"samples": n,
                          "meter_ms": round(device_ms(lambda: loudness.meter(wav, 16000, [n]), it, wu), 4),
                          "model_meter_ms": round(device_ms(lambda: model.meter(out), it, wu), 4),
                          "format_float32_ms": round(device_ms(lambda: model.format_audio(out, 16000, "float32"), it, wu), 4)}}
    print("b1_fixture", json.dumps(rec["b1_fixture"]), flush=True)
    w32 = torch.from_numpy((0.1 * np.random.default_rng(32).standard_normal((32, 160000))).astype(np.float32)).to(dev)
    rec["b32_10s_16k"] = {"meter_ms": round(device_ms(lambda: loudness.meter(w32, 16000), it, wu), 4),
                          "meter_series_ms": round(device_ms(lambda: loudness.meter(w32, 16000, series=True), it, wu), 4)}
    print("b32_10s_16k", json.dumps(rec["b32_10s_16k"]), flush=True)
    sr = 48000
    hour = torch.from_numpy((0.1 * np.random.default_rng(60).standard_normal((1, 3600 * sr))).astype(np.float32)).to(dev)
    rec["one_hour_48k"] = {"samples": 3600 * sr,
                           "meter_ms": round(device_ms(lambda: loudness.meter(hour, sr), max(3, it // 10), 2), 3),
                           "meter_series_ms": round(device_ms(lambda: loudness.meter(hour, sr, series=True), max(3, it // 10), 2), 3)}
    print("one_hour_48k", json.dumps(rec["one_hour_48k"]), flush=True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        loudness.meter(hour, sr)
        torch.cuda.synchronize()
    rec["one_hour_48k"]["kernel_ms"] = {e.key: round(e.device_time_total / 1000.0, 3) for e in prof.key_averages()
                                        if e.device_time_total > 0}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), iters=args.iters, warmup=args.warmup, **rec)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
