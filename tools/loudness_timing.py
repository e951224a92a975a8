"""Times loudness normalisation on the GPU (JETSGenerator.format_audio with and without ``loudness``: ev_loudness's two
launches ahead of the format launch) against the host path a server would otherwise run on the same outputs.

Workloads: the b1_t100 fixture's 537-frame utterance at B=1 (137,472 samples), and a cfg3-like batch (B=32, 20..200 phonemes,
the lengths of tools/audio_format_timing.py), each at 8 kHz mu-law and 24 kHz pcm16.  GPU: CUDA events around --iters
format_audio calls after --warmup, mean per call on the device timeline (the offsets' H2D copy + the launches; the waveform is
already on the device).  Host: a device->host copy of the valid fp32 samples (fetch_audio at 16 kHz float32), then per item
K-weighting with scipy.signal.lfilter, gating, the gain, resample_poly and the encoding (the fp64 oracle's routines), mean of
--cpu-iters runs, one thread (the numpy / scipy defaults), summed over the batch.

    python tools/loudness_timing.py [--iters 200] [--warmup 20] [--cpu-iters 5] [--out profiles/h100_loudness_timing.json]

Reads the GPU name and power limit in the same run; prints the record and writes it to --out."""
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

from emotivoice_b200 import audio, synth                    # noqa: E402
from emotivoice_b200 import frontdoor as fd                 # noqa: E402
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402
from oracle import loudness_oracle as O                     # noqa: E402

FORMATS = [(8000, "mulaw"), (24000, "pcm16")]
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
TARGET = -23.0


def host_normalise(x, rate, encoding, ulaw):
    from scipy.signal import resample_poly
    L = O.integrated_loudness(x, 16000)
    g = O.gain(L, O.peak(x), TARGET)
    _, up, down = audio.plan(rate, encoding, 16000)
    y = resample_poly(x * g, up, down)
    pcm = np.clip(np.trunc(y * 32768.0), -32768, 32767).astype(np.int16)
    return ulaw[pcm.astype(np.int64) + 32768] if encoding == "mulaw" else pcm


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
    ap.add_argument("--cpu-iters", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_loudness_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the loudness kernels run on the GPU only")
    dev = torch.device("cuda:0")
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    ulaw = np.load(os.path.join(ROOT, "tests", "golden", "g711.npz"))["ulaw"]
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
        lufs, _ = model.measure_loudness(out)
        res[name] = {"batch": len(n_in), "samples_in": sum(n_in), "lufs": [round(float(v), 3) for v in lufs.cpu().tolist()]}
        for rate, enc in FORMATS:
            plain_ms = device_ms(lambda: model.format_audio(out, rate, enc), args.iters, args.warmup)
            loud_ms = device_ms(lambda: model.format_audio(out, rate, enc, loudness=TARGET), args.iters, args.warmup)
            host_ms = []
            for _ in range(args.cpu_iters):
                t0 = time.perf_counter()
                xs = fd.fetch_audio(model, out, None, "float32")
                t1 = time.perf_counter()
                for x in xs:
                    host_normalise(x.astype(np.float64), rate, enc, ulaw)
                host_ms.append(((t1 - t0) * 1e3, (time.perf_counter() - t1) * 1e3))
            d2h, cpu = np.mean(host_ms, axis=0)
            r = {"gpu_ms_per_call": round(plain_ms, 4), "gpu_ms_per_call_loudness": round(loud_ms, 4),
                 "loudness_extra_ms": round(loud_ms - plain_ms, 4), "host_d2h_ms": round(float(d2h), 3),
                 "host_normalise_encode_ms": round(float(cpu), 3)}
            res[name]["%d_%s" % (rate, enc)] = r
            print(name, rate, enc, json.dumps(r), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), cpu=os.cpu_count(), target_lufs=TARGET, iters=args.iters, warmup=args.warmup,
               cpu_iters=args.cpu_iters, results=res)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
