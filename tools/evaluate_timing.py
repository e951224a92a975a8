"""Times the comparison of syntheses with recordings on the GPU (``evaluate.compare``; ``ev_eval_compare``: three launches).

Cases, at 16 kHz, each synthesis against a recording 8 % longer (so N != M):
- one_10s: one pair of 10 s.
- b32_10s: 32 pairs of 10 s.
- one_65s: one pair at the length limit (4096 frames on the longer side).
For each: ``compare`` end to end (log-mel and F0 of both sides, then ev_eval_compare) and ev_eval_compare alone on those
features, CUDA events around --iters calls after --warmup, mean per call on the device timeline.  The per-kernel device times
of b32_10s come from torch.profiler in a run of their own.  For scale, ``oracle/eval_oracle.py`` (numpy fp64 on the host CPU,
one pair at a time) on the same features, labelled as the CPU fp64 oracle.

    python tools/evaluate_timing.py [--iters 20] [--warmup 3] [--out profiles/h100_evaluate_timing.json]

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

from emotivoice_b200 import _abi, evaluate                  # noqa: E402
from oracle import eval_oracle                              # noqa: E402

SR = 16000


def voiced(seconds, seed):
    """A seeded harmonic signal with a gliding F0, amplitude-modulated into syllables, over a low noise floor."""
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    t = np.arange(n) / SR
    f0 = 150.0 + 40.0 * np.sin(2 * np.pi * 0.3 * t + rng.uniform(0, 6.28))
    ph = 2 * np.pi * np.cumsum(f0) / SR
    x = sum(np.sin(h * ph) / h for h in range(1, 30))
    x *= np.clip(np.sin(2 * np.pi * 2.5 * t + rng.uniform(0, 6.28)), 0.0, None)
    x = 0.3 * x / np.abs(x).max() + 1e-3 * rng.standard_normal(n)
    return x.astype(np.float32)


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


def abi_call(lib, dev, ms, fs, ns, mr, fr, nr):
    """ev_eval_compare on ready features -> a closure that enqueues it once."""
    B = len(ns)
    cnt = torch.tensor(ns + nr, dtype=torch.int32, device=dev)
    stats = torch.empty((3, B), dtype=torch.float64, device=dev)
    counts = torch.empty((2, B), dtype=torch.int32, device=dev)
    nb = int(lib.ev_eval_workspace_bytes(B, max(ns), max(nr)))
    ws = torch.empty((nb,), dtype=torch.uint8, device=dev)
    table = torch.from_numpy(evaluate.cos_table()).to(dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def run():
        _abi.check(lib.ev_eval_compare(ms.data_ptr(), fs.data_ptr(), ms.shape[2], cnt.data_ptr(), max(ns), mr.data_ptr(), fr.data_ptr(),
                                       mr.shape[2], cnt.data_ptr() + 4 * B, max(nr), B, table.data_ptr(), stats.data_ptr(),
                                       counts.data_ptr(), None, 0, ws.data_ptr(), nb, st))
    return run, nb


def case(lib, dev, B, seconds, iters, warmup, oracle_pairs):
    syn = [voiced(seconds, 2 * b) for b in range(B)]
    ref = [voiced(seconds * 1.08, 2 * b + 1)[:4096 * 256 - 1] for b in range(B)]
    ws_, wr = (torch.from_numpy(np.stack(x)).to(dev) for x in (syn, ref))
    ls, lr = [len(syn[0])] * B, [len(ref[0])] * B
    rec = {"pairs": B, "syn_samples": ls[0], "ref_samples": lr[0], "syn_frames": ls[0] // 256 + 1, "ref_frames": lr[0] // 256 + 1}
    rec["compare_ms"] = round(device_ms(lambda: evaluate.compare(ws_, wr), iters, warmup), 3)
    ms, fs = evaluate._features(ws_, ls)
    mr, fr = evaluate._features(wr, lr)
    ns, nr = [rec["syn_frames"]] * B, [rec["ref_frames"]] * B
    run, nb = abi_call(lib, dev, ms, fs, ns, mr, fr, nr)
    rec["ev_eval_compare_ms"] = round(device_ms(run, iters, warmup), 3)
    rec["workspace_bytes"] = nb
    rec["cells"] = B * ns[0] * nr[0]
    h = [t.cpu().numpy() for t in (ms, fs, mr, fr)]
    t0 = time.perf_counter()
    for b in range(oracle_pairs):
        eval_oracle.compare(h[0][b, :, :ns[b]], h[1][b, :ns[b]], h[2][b, :, :nr[b]], h[3][b, :nr[b]])
    rec["cpu_fp64_oracle_s_per_pair"] = round((time.perf_counter() - t0) / oracle_pairs, 3)
    return rec, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_evaluate_timing.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: the comparison kernels run on the GPU only")
    dev = torch.device("cuda:0")
    lib = _abi.load()
    rec = {}
    for name, B, seconds, oracle_pairs in (("one_10s", 1, 10.0, 1), ("b32_10s", 32, 10.0, 4), ("one_65s", 1, 4096 * 256 / 1.08 / SR, 1)):
        rec[name], run = case(lib, dev, B, seconds, args.iters, args.warmup, oracle_pairs)
        print(name, json.dumps(rec[name]), flush=True)
        if name == "b32_10s":
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            rec[name]["kernel_ms"] = {e.key: round(e.device_time_total / 1000.0, 3) for e in prof.key_averages()
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
