"""Times a phoneme-controlled forward against a plain one and a per-item-controlled one (CUDA events, B=1 and B=8 at 100
phonemes, seeded weights), with the number of library launches each enqueues.

    python tools/token_prosody_timing.py [--iters 50]

Prints one JSON line with the GPU name, its power limit and the median milliseconds per forward of each variant."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from emotivoice_b200 import _abi, synth                       # noqa: E402
from emotivoice_b200.config import default_config            # noqa: E402
from emotivoice_b200.modules import JETSGenerator            # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    conf = default_config()
    m = JETSGenerator(conf).to(dev).eval()
    m.load_state_dict(synth.make_state_dict(conf))
    res = {}
    for B in (1, 8):
        batch = {k: v.to(dev) for k, v in synth.make_batch([100] * B).items()}
        T = int(batch["inputs_ling"].shape[1])
        plain = m(**batch)
        rate = np.where(np.arange(T) % 7 == 3, 1.5, 0.9)[None, :].repeat(B, 0)
        variants = {
            "plain": {},
            "per_item": dict(duration_scale=[0.9] * B, pitch_shift=[2.0] * B),
            "per_token": dict(duration_scale=rate, pitch_shift=np.where(np.arange(T) < 30, 3.0, 0.0)[None, :].repeat(B, 0)),
            "caller_values": dict(durations=plain["log_duration_predictions"], pitch=plain["pitch_predictions"], duration_scale=rate),
        }
        for name, kw in variants.items():
            for _ in range(3):
                m(**batch, **kw)
            torch.cuda.synchronize()
            n0 = _abi.launch_count()
            m(**batch, **kw)
            torch.cuda.synchronize()
            launches = _abi.launch_count() - n0
            times = []
            for _ in range(args.iters):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                m(**batch, **kw)
                e.record()
                e.synchronize()
                times.append(s.elapsed_time(e))
            res["B%d_%s" % (B, name)] = dict(ms_median=float(np.median(times)), launches=launches)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(gpu=q.stdout.strip(), results=res)))


if __name__ == "__main__":
    main()
