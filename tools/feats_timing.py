"""Times the fused log-mel + energy kernel (stft_feats_kernel, one ev_stft_features launch at the config: 16 kHz, hop 256, 80 mels,
TacotronSTFT's padding and window) against the same math through torch on the same GPU (torch.stft + magnitude + mel matmul +
log, and the energy sum) and against the reference's conv1d form (oracle/feats_oracle.py: tacotron_mel) on the host CPU.

Workloads: B=1 on the b1_t100 fixture's 8.6 s waveform; B=32 items of 1-10 s (seeded), padded to the longest with per-item
lengths.  GPU: CUDA events around --iters calls after --warmup, mean per call on the device timeline.  CPU: the mean of
--cpu-iters calls, per item, summed over the batch.  The kernel's HBM traffic is counted as the samples it reads (each tile's
span once) plus the mel and energy it writes; over the data sheet's 3.35 TB/s that gives the achieved fraction.

    python tools/feats_timing.py [--iters 200] [--warmup 20] [--cpu-iters 2] [--out FILE]

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
from oracle import feats_oracle as FO                       # noqa: E402

SR, HOP, N_MELS, HBM_BPS = 16000, 256, 80, 3.35e12
TILE = 32                                                   # frames per CTA of stft_feats_kernel


def kernel_bytes(lens, N):
    F = feats.n_frames(N, 512, HOP)
    read = 0
    for n in lens:
        fb = feats.n_frames(n, 512, HOP)
        for f0 in range(0, fb, TILE):
            read += HOP * (min(TILE, fb - f0) - 1) + 1024
    return 4 * read + 4 * len(lens) * F * (N_MELS + 1)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--cpu-iters", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the feature kernel runs on the GPU only")
    dev = torch.device("cuda:0")
    with np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz")) as z:
        b1 = z["wav"].reshape(-1).astype(np.float32)
    rng = np.random.default_rng(3232)
    lens = rng.integers(1 * SR, 10 * SR + 1, size=32).tolist()
    items = [(0.3 * rng.standard_normal(n)).clip(-1, 1).astype(np.float32) for n in lens]
    workloads = {"b1_fixture": ([b1], None), "b32_1to10s": (items, lens)}
    stft = feats.TacotronSTFT(sampling_rate=SR).to(dev)
    bands = feats.device_bands(stft.mel_basis, dev)
    basis = stft.mel_basis
    win = torch.hann_window(1024, device=dev)
    res = {}
    for name, (its, ls) in workloads.items():
        N = max(len(x) for x in its)
        y = torch.zeros(len(its), N)
        for b, x in enumerate(its):
            y[b, :len(x)] = torch.from_numpy(x)
        y = y.to(dev)
        lens_b = [len(x) for x in its]
        frames = sum(feats.n_frames(n, 512, HOP) for n in lens_b)

        def kernel():
            return feats.stft_features(y, 512, HOP, stft.window, 0.0, bands=bands, energy=True, lengths=ls)

        def torch_path():
            spec = torch.stft(y, 1024, hop_length=HOP, win_length=1024, window=win, center=True, pad_mode="reflect", return_complex=True)
            p = spec.real ** 2 + spec.imag ** 2
            mel = torch.log(torch.clamp(torch.matmul(basis, torch.sqrt(p)), min=1e-5))
            return mel, torch.sqrt(torch.clamp(p.sum(1), min=1e-10))

        k_ms = timed(kernel, args.iters, args.warmup)
        t_ms = timed(torch_path, args.iters, args.warmup)
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            with torch.no_grad():
                for x in its:
                    FO.tacotron_mel(x, HOP)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        nbytes = kernel_bytes(lens_b, N)
        mel_k = kernel()[0]
        mel_t = torch_path()[0]
        # frames whose window ends inside the item: past them torch.stft reflects the batch's zero padding, the kernel the item
        diff = max(float((mel_k[b, :, :(n - 512) // HOP + 1] - mel_t[b, :, :(n - 512) // HOP + 1]).abs().max()) for b, n in enumerate(lens_b))
        res[name] = {"batch": len(its), "samples": sum(lens_b), "frames": frames, "kernel_ms": round(k_ms, 4),
                     "torch_gpu_ms": round(t_ms, 4), "reference_conv1d_cpu_ms": round(cpu_ms, 2), "kernel_bytes": nbytes,
                     "kernel_hbm_fraction": round(nbytes / (k_ms * 1e-3) / HBM_BPS, 4), "max_abs_logmel_diff_vs_torch": diff}
        print(name, json.dumps(res[name]), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    line = json.dumps(dict(gpu=q.stdout.strip(), cpu=os.cpu_count(), iters=args.iters, warmup=args.warmup, cpu_iters=args.cpu_iters,
                           hbm_peak_bytes_per_s=HBM_BPS, results=res))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
