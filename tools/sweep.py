"""cfg3 (batch-32 mixed lengths) and cfg4 (vocoder-only sweep) measurements (BASELINE.json configs[2], [3]).

    python tools/sweep.py [--out profiles/r01_sweep.json]

Vocoder roofline accounting (SURVEY.md s8d): 614,105,088 FLOP and 5,010,752 B (layer-granular fp32
activation traffic) per mel frame; reported as achieved TFLOP/s, GB/s and fractions of the measured peaks."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from emotivoice_b200 import build, synth
from emotivoice_b200.config import default_config
from emotivoice_b200.modules import JETSGenerator

FLOP_PER_FRAME = 614105088.0
BYTES_PER_FRAME = 5010752.0


def timed(fn, reps, flush):
    ts = []
    for i in range(reps + 2):
        flush()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        if i >= 2:
            ts.append(e0.elapsed_time(e1) * 1e-3)
    return statistics.median(ts), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--corner", action="store_true", help="add the B=64, F=4096 corner of cfg4 (the largest that fits 80 GB)")
    ap.add_argument("--no-cfg3", action="store_true")
    ap.add_argument("--precisions", default="fp32,tf32", help="comma separated: fp32,tf32,bf16")
    args = ap.parse_args()
    precisions = tuple(args.precisions.split(","))
    build.build(verbose=False)
    peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(
        os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"hbm_gbs": 6650.0, "bf16_tflops": 1590.0}
    dev = torch.device("cuda:0")
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    flush_buf = torch.empty(64 * 1024 * 1024, device=dev)
    flush = flush_buf.zero_
    res = {"peaks": peaks, "env": {k: v for k, v in os.environ.items() if k.startswith("EV_")}, "cfg3": {}, "cfg4": []}

    # ---- cfg3: batch 32, 20..200 phonemes -------------------------------------------------
    import numpy as np
    rng = np.random.default_rng(32)
    lens = sorted(rng.integers(20, 201, size=32).tolist(), reverse=True)
    batch = {k: v.to(dev) for k, v in synth.make_batch(lens, seed=3232).items()}
    for prec in ([] if args.no_cfg3 else precisions):
        model.precision = prec
        t, out = timed(lambda: model(**batch), 5, flush)
        frames = int(out["mel_lengths"].sum())
        res["cfg3"][prec] = {"batch": 32, "phonemes": lens, "frames_valid": frames, "frames_padded": int(32 * out["dec_outputs"].shape[1]),
                            "seconds": t, "mel_frames_per_sec": frames / t, "x_realtime": frames * 256 / 16000 / t}
        # batch-invariance spot check against B=1 runs (bitwise)
        ok = True
        for b in (0, 17, 31):
            single = model(**{k: v.to(dev) for k, v in synth.slice_batch({k: v.cpu() for k, v in batch.items()}, b).items()})
            Fb = single["dec_outputs"].shape[1]
            ok = ok and torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256])
        res["cfg3"][prec]["bitwise_equal_to_b1_runs"] = bool(ok)
        print("cfg3", prec, json.dumps({k: v for k, v in res["cfg3"][prec].items() if k != "phonemes"}), flush=True)

    # ---- cfg4: vocoder-only sweep ------------------------------------------------------------
    points = [(1, 256), (1, 1024), (1, 4096), (8, 1024), (32, 1024)] if args.quick else \
        [(1, 256), (1, 512), (1, 1024), (1, 2048), (1, 4096), (4, 1024), (8, 1024), (16, 1024), (32, 512), (32, 1024), (64, 512), (128, 256)]
    if args.corner:
        points = points + [(64, 4096)]           # the largest point of BASELINE.json configs[3] that fits 80 GB: 47 GB of vocoder workspace in the fp32-storage modes
    for prec in precisions:
        model.precision = prec
        for B, F in points:
            mel = synth.make_mel(B, F, seed=B * 7 + F).to(dev)
            try:
                t, _ = timed(lambda: model.generator(mel), 2 if B * F > 100000 else 3, flush)
            except Exception as e:          # an out-of-memory at the corner must not cost the other points
                print("cfg4", json.dumps({"precision": prec, "batch": B, "frames": F, "error": repr(e)[:200]}), flush=True)
                torch.cuda.empty_cache()
                continue
            fr = B * F
            # note: model.generator is the stand-alone Generator module (its own engine, fp32 precision attr set below)
            row = {"precision": prec, "batch": B, "frames": F, "seconds": t, "mel_frames_per_sec": fr / t,
                   "tflops_algorithmic": fr * FLOP_PER_FRAME / t / 1e12, "gbs_layer_granular": fr * BYTES_PER_FRAME / t / 1e9,
                   "frac_hbm": fr * BYTES_PER_FRAME / t / 1e9 / peaks["hbm_gbs"],
                   "frac_tensor_bf16_peak": fr * FLOP_PER_FRAME / t / 1e12 / peaks["bf16_tflops"]}
            res["cfg4"].append(row)
            print("cfg4", json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
