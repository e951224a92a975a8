"""Times FLAC output on the GPU: ev_flac_encode alone (CUDA events), and fetch_audio end to end with encoding="flac" against
"pcm16" (host clock around each call, which ends in a synchronise; the flac call includes its read of the image offsets), and
reports the bytes against PCM16.

Workloads: the b1_t100 fixture's 537-frame utterance at B=1 (8.6 s at 16 kHz), at 16 and 48 kHz; and B=32 engine outputs of
1-10 s (a seeded batch of 8..75 phonemes; the durations are recorded).  Compression ratios are also reported for the
synthetic signals of tests/test_flac.py.  With seeded random weights the engine's waveform is not speech, so its ratio says
little about a trained checkpoint.  The numpy oracle's host time for the B=1 item is listed, labelled as the oracle: it is not
a libFLAC baseline.

    python tools/flac_timing.py [--iters 200] [--warmup 20] [--out profiles/h100_flac_timing.json]

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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from emotivoice_b200 import _abi, synth                     # noqa: E402
from emotivoice_b200 import frontdoor as fd                 # noqa: E402
from emotivoice_b200.config import default_config           # noqa: E402
from emotivoice_b200.modules import JETSGenerator           # noqa: E402
from oracle import flac_oracle as F                         # noqa: E402

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


def host_ms(fns, iters, warmup):
    """Alternating host-clock means of each fn (each ends in a synchronise)."""
    for _ in range(warmup):
        for f in fns:
            f()
    t = np.zeros(len(fns))
    for _ in range(iters):
        for i, f in enumerate(fns):
            t0 = time.perf_counter()
            f()
            t[i] += time.perf_counter() - t0
    return (t / iters * 1e3).tolist()


class Encoder:
    """ev_flac_encode on fixed int16 items with preallocated buffers."""

    def __init__(self, lib, dev, pcm, offs, rate):
        self.lib, self.rate = lib, rate
        self.counts = np.ascontiguousarray(np.diff(offs), dtype=np.int64)
        self.pcm, self.pcm_off = pcm, torch.from_numpy(offs).to(dev)
        self.bound = sum(int(lib.ev_flac_bound_bytes(int(n))) for n in self.counts)
        self.out = torch.empty(self.bound, dtype=torch.uint8, device=dev)
        self.out_off = torch.empty(len(self.counts) + 1, dtype=torch.int64, device=dev)
        self.nb = lib.ev_flac_workspace_bytes(len(self.counts), int(self.counts.max()))
        self.ws = torch.empty(self.nb, dtype=torch.uint8, device=dev)
        self.st = torch.cuda.current_stream(dev).cuda_stream

    def __call__(self):
        _abi.check(self.lib.ev_flac_encode(self.pcm.data_ptr(), self.pcm_off.data_ptr(), len(self.counts), self.counts.ctypes.data,
                                           self.rate, self.out.data_ptr(), self.bound, self.out_off.data_ptr(), self.ws.data_ptr(),
                                           self.nb, self.st))

    def sizes(self):
        return np.diff(self.out_off.cpu().numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_flac_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the FLAC kernels run on the GPU only")
    dev = torch.device("cuda:0")
    lib = _abi.load()
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    g = np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz"))
    rng = np.random.default_rng(32)
    lens = sorted(rng.integers(8, 76, size=32).tolist(), reverse=True)
    workloads = {"b1_fixture": {k: torch.from_numpy(g[k]).to(dev) for k in KEYS},
                 "b32": {k: v.to(dev) for k, v in synth.make_batch(lens, seed=3232).items()}}
    res = {}
    for name, batch in workloads.items():
        out = model(**batch)
        torch.cuda.synchronize()
        secs = [round(int(n) * 256 / 16000, 2) for n in out["mel_lengths_host"].tolist()]
        for rate in ((16000, 48000) if name == "b1_fixture" else (16000,)):
            pcm, offs = model.format_audio(out, rate, "pcm16")
            enc = Encoder(lib, dev, pcm, offs, rate)
            kernel_ms = device_ms(enc, args.iters, args.warmup)
            flac_bytes, pcm_bytes = int(enc.sizes().sum()), 2 * int(offs[-1])
            e2e_flac, e2e_pcm = host_ms([lambda: fd.fetch_audio(model, out, rate, "flac"), lambda: fd.fetch_audio(model, out, rate, "pcm16")],
                                        max(args.iters // 4, 10), 5)
            r = {"batch": len(secs), "seconds": [min(secs), max(secs), round(sum(secs), 2)], "samples": int(offs[-1]),
                 "ev_flac_encode_device_ms": round(kernel_ms, 4), "fetch_audio_flac_ms": round(e2e_flac, 4),
                 "fetch_audio_pcm16_ms": round(e2e_pcm, 4), "flac_bytes": flac_bytes, "pcm16_bytes": pcm_bytes,
                 "flac_over_pcm16": round(flac_bytes / pcm_bytes, 4)}
            if name == "b1_fixture" and rate == 16000:
                x = fd.fetch_audio(model, out, rate, "pcm16")[0]
                t0 = time.perf_counter()
                F.encode(x, rate)
                r["numpy_oracle_encode_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            res["%s_%d" % (name, rate)] = r
            print(name, rate, json.dumps(r), flush=True)
    from test_flac import signals
    sig = signals()
    ratios = {}
    for k, x in sig.items():
        pcm = torch.from_numpy(x).to(dev)
        enc = Encoder(lib, dev, pcm, np.array([0, len(x)], np.int64), 16000)
        enc()
        ratios[k] = round(float(enc.sizes()[0]) / (2 * len(x)), 4)
    res["synthetic_flac_over_pcm16"] = ratios
    print("synthetic", json.dumps(ratios))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rec = dict(gpu=q.stdout.strip(), cpu=os.cpu_count(), iters=args.iters, warmup=args.warmup, results=res)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
