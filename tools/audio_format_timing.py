"""Times the output formatting (JETSGenerator.format_audio, one ev_format_audio launch) on the GPU against the host conversion a
server would otherwise run (scipy.signal.resample_poly of the float32 waveform + cast to int16 + G.711 table lookup) on this
machine's CPU.

Workloads: the b1_t100 fixture's 537-frame utterance at B=1 (137,472 samples), and a cfg3-like batch (B=32, 20..200 phonemes,
the lengths of tools/sweep.py), each at 8 kHz mu-law, 24 kHz pcm16, 44.1 kHz pcm16 and 48 kHz pcm16.  GPU: CUDA events around
--iters format_audio calls after --warmup, mean per call on the device timeline (the offsets' H2D copy + the kernel; the
waveform is already on the device).  CPU: the mean of
--cpu-iters calls of resample_poly + cast per item, one thread (the numpy / scipy defaults), summed over the batch.

    python tools/audio_format_timing.py [--iters 200] [--warmup 20] [--cpu-iters 5]

Prints one JSON line with the GPU name and power limit (read in the same run)."""
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
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402

FORMATS = [(8000, "mulaw"), (24000, "pcm16"), (44100, "pcm16"), (48000, "pcm16")]
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")


def host_convert(x, rate, encoding, ulaw):
    from scipy.signal import resample_poly
    _, up, down = audio.plan(rate, encoding, 16000)
    y = resample_poly(x, up, down) if (up, down) != (1, 1) else x
    pcm = np.clip(np.trunc(y * 32768.0), -32768, 32767).astype(np.int16)
    return ulaw[pcm.astype(np.int64) + 32768] if encoding == "mulaw" else pcm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--cpu-iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the format kernel runs on the GPU only")
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
        wav = out["wav_predictions"].cpu().numpy()
        items = [wav[b, 0, :n] for b, n in enumerate(n_in)]
        res[name] = {"batch": len(n_in), "samples_in": sum(n_in), "padded_samples": int(out["wav_predictions"].numel())}
        for rate, enc in FORMATS:
            for _ in range(args.warmup):
                model.format_audio(out, rate, enc)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.iters):
                packed, _ = model.format_audio(out, rate, enc)
            e.record()
            torch.cuda.synchronize()
            gpu_ms = s.elapsed_time(e) / args.iters
            t0 = time.perf_counter()
            for _ in range(args.cpu_iters):
                for x in items:
                    host_convert(x, rate, enc, ulaw)
            cpu_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
            res[name]["%d_%s" % (rate, enc)] = {"samples_out": int(packed.numel()), "gpu_ms_per_call": round(gpu_ms, 4),
                                                 "host_resample_cast_ms": round(cpu_ms, 3)}
            print(name, rate, enc, json.dumps(res[name]["%d_%s" % (rate, enc)]), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(gpu=q.stdout.strip(), cpu=os.cpu_count(), iters=args.iters, warmup=args.warmup, cpu_iters=args.cpu_iters,
                          results=res)))


if __name__ == "__main__":
    main()
