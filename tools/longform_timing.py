"""Times a ~1,000-phoneme paragraph two ways: as one utterance, and split at pause tokens (frontdoor.split_phonemes,
max_phonemes=256) into segments run as one batch whose mel is joined and vocoded as one waveform (forward(join=...)).
CUDA events after warm-up, fp32 and bf16, seeded weights; the paragraph is lines 1-10 of the reference's inference text
(tests/golden/frontdoor/inference_text), their inner tokens between one pair of <sos/eos>.

    python tools/longform_timing.py [--iters 10] [--warmup 3]

Prints one JSON line with the GPU name and power limit (read in the same run) and, per precision and variant, the median
milliseconds per forward, the frames synthesised and the segment lengths."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200 import frontdoor as fd, synth             # noqa: E402
from emotivoice_b200.config import default_config            # noqa: E402
from emotivoice_b200.modules import JETSGenerator            # noqa: E402

FRONTDOOR = os.path.join(ROOT, "tests", "golden", "frontdoor")


def paragraph():
    with open(os.path.join(FRONTDOOR, "inference_text"), encoding="utf-8") as f:
        lines = [fd.parse_line(l).phonemes for l in f if l.strip()]
    return [fd.SOS_EOS] + [t for toks in lines[:10] for t in toks[1:-1]] + [fd.SOS_EOS]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("longform_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    conf = default_config()
    m = JETSGenerator(conf).to(dev).eval()
    m.load_state_dict(synth.make_state_dict(conf))
    t2i = fd.load_symbol_table(os.path.join(FRONTDOOR, "tokenlist"))
    rng = np.random.default_rng(7)
    style, content = (np.tanh(rng.normal(size=768)).astype(np.float32) for _ in range(2))
    para = paragraph()
    segs = fd.split_phonemes(para, max_phonemes=256)

    def batch_of(seqs):
        b = fd.collate([(np.asarray([t2i[p] for p in s], dtype=np.int64), 0, style, content) for s in seqs])
        return {k: v.to(dev) for k, v in b.items()}
    variants = {"one_utterance": (batch_of([para]), {}),
                "joined_256": (batch_of(segs), dict(join=[0] * len(segs)))}
    res = dict(phonemes=len(para), segments=[len(s) for s in segs])
    for precision in ("fp32", "bf16"):
        m.precision = precision
        for name, (batch, kw) in variants.items():
            for _ in range(args.warmup):
                out = m(**batch, **kw)
            torch.cuda.synchronize()
            frames = int(out["joined_lengths_host"][0]) if "join" in kw else int(out["mel_lengths_host"][0])
            times = []
            for _ in range(args.iters):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                m(**batch, **kw)
                e.record()
                e.synchronize()
                times.append(s.elapsed_time(e))
            res["%s_%s" % (precision, name)] = dict(ms_median=float(np.median(times)), ms_min=float(np.min(times)), frames=frames)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(gpu=q.stdout.strip(), iters=args.iters, results=res)))


if __name__ == "__main__":
    main()
