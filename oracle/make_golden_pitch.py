"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/pitch_*.npz from the reference's own ``feats.Pitch``
(models/prompt_tts_modified/feats.py:83-156).  Run where the reference tree is present:  python oracle/make_golden_pitch.py

The unmodified class is imported with make_golden_feats' stub ``librosa`` / ``pyworld`` modules, and the ``pyworld`` stub is
given oracle/pitch_oracle.py's ``dio`` and ``stonemask`` (a restatement, not pyworld).  So the reference's own glue runs as
written: ``_convert_to_continuous_pitch``, the log and ``_average_by_duration``.  The oracle's restatement of that glue is
checked here against it, bit for bit.

Signals (each over a -80 dBFS Gaussian noise floor, so no voicing decision rests on round-off), at 16 kHz / hop 256 unless
named otherwise: stationary harmonic complexes at 90, 150, 220 and 330 Hz; 180 Hz with 5 Hz, +-4 % vibrato; an exponential
80 -> 400 Hz glide; 180 Hz alternating with -30 dBFS noise every 0.3 s; noise alone (the all-zero early return); the excerpt of
tests/golden/b1_t100.npz's waveform that feats_b1_t100.npz uses; and a 250 Hz complex with vibrato at the class default of
24 kHz / hop 300.  Each fixture holds the float32 input, DIO's contour, the refined contour, the continuous, log and
continuous-log tracks, token averages over seeded durations, and the known F0 per frame (0 where there is none).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_feats as MGF   # noqa: E402
from oracle import pitch_oracle as PO         # noqa: E402
from oracle import refshim                    # noqa: E402

FLOOR = 1e-4                                   # -80 dBFS rms


def _complex(phase, amp=0.3, n_harm=5):
    return sum(amp / k * np.sin(k * phase + 0.7 * k) for k in range(1, n_harm + 1))


def signals():
    """name -> (wav float32, sr, hop, known F0 as a function of time in s (0: none))."""
    rng = np.random.default_rng(9700)
    out = {}

    def put(name, sr, dur, f_of_t, voiced=None, extra=None):
        t = np.arange(int(dur * sr)) / sr
        f = f_of_t(t)
        phase = 2 * np.pi * np.cumsum(f) / sr
        y = _complex(phase)
        if voiced is not None:
            y = y * voiced(t)
        if extra is not None:
            y = y + extra(t)
        y = y + FLOOR * rng.standard_normal(len(t))
        known = (lambda tt, f_of_t=f_of_t, voiced=voiced: f_of_t(tt) * (1.0 if voiced is None else voiced(tt)))
        out[name] = (y.astype(np.float32), sr, 256 if sr == 16000 else 300, known)

    for f0 in (90.0, 150.0, 220.0, 330.0):
        put("stat%d" % int(f0), 16000, 0.8, lambda t, f0=f0: np.full_like(t, f0))
    put("vibrato", 16000, 1.5, lambda t: 180.0 * (1 + 0.04 * np.sin(2 * np.pi * 5 * t)))
    put("glide", 16000, 2.0, lambda t: 80.0 * 5.0 ** (t / 2.0))
    gate = lambda t: (np.floor(t / 0.3) % 2 == 0).astype(np.float64)         # noqa: E731
    put("alternate", 16000, 1.8, lambda t: np.full_like(t, 180.0), voiced=gate,
        extra=lambda t: 0.0316 * (1 - gate(t)) * np.random.default_rng(9701).standard_normal(len(t)))
    n = int(0.8 * 16000)
    out["noise"] = ((FLOOR * rng.standard_normal(n)).astype(np.float32), 16000, 256, lambda tt: np.zeros_like(tt))
    wav = np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz"))["wav"].reshape(-1)
    out["b1_t100"] = (wav[MGF.B1_SPAN[0]:MGF.B1_SPAN[1]].astype(np.float32), 16000, 256, None)
    put("sr24k", 24000, 1.0, lambda t: 250.0 * (1 + 0.03 * np.sin(2 * np.pi * 4 * t)))
    return out


def durations(F, seed):
    rng = np.random.default_rng(seed)
    d = []
    while sum(d) < F:
        d.append(int(rng.integers(0, 9)))
    d[-1] -= sum(d) - F
    return np.asarray(d, np.int64)


def main():
    if not refshim.reference_available():
        raise SystemExit("reference tree not present at %s" % refshim.REF_ROOT)
    MGF.install_stubs()
    pw = sys.modules["pyworld"]
    pw.dio, pw.stonemask = PO.dio, PO.stonemask
    if refshim.REF_ROOT not in sys.path:
        sys.path.insert(0, refshim.REF_ROOT)
    from models.prompt_tts_modified import feats as RF
    out_dir = os.path.join(ROOT, "tests", "golden")
    for k, (name, (y, sr, hop, known)) in enumerate(signals().items()):
        x = y.astype(np.float64)
        P = RF.Pitch(sr=sr, hop_length=hop)
        fp = 1000 * hop / sr
        f0, t = PO.dio(x, sr, fp)
        ref = PO.stonemask(x, f0, t, sr)
        F = len(f0)
        assert F == PO.frame_count(len(x), sr, fp) == len(x) // hop + 1, name
        cont = P.get_pitch(y, use_continuous_pitch=True)
        raw = P.get_pitch(y, use_continuous_pitch=False)
        lg = P.get_pitch(y, use_continuous_pitch=True, use_log_pitch=True)
        lg_nc = P.get_pitch(y, use_continuous_pitch=False, use_log_pitch=True)
        d = durations(F, 9800 + k)
        tok = P.get_pitch(y, use_token_averaged_pitch=True, duration=d)
        assert np.array_equal(raw, ref), name
        assert np.array_equal(PO.continuous(ref), cont), name
        assert np.array_equal(PO.log_pitch(PO.continuous(ref)), lg), name
        assert np.array_equal(PO.log_pitch(ref), lg_nc), name
        assert np.array_equal(PO.average_by_duration(cont, d), tok), name
        arrays = {"wav": y, "sr": np.int64(sr), "hop": np.int64(hop), "f0_dio": f0, "f0_refined": ref, "continuous": cont,
                  "log": lg, "log_raw": lg_nc, "durations": d, "token_avg": np.asarray(tok, np.float64)}
        if known is not None:
            arrays["known_f0"] = known(t)
        np.savez_compressed(os.path.join(out_dir, "pitch_%s.npz" % name), **arrays)
        v = ref > 0
        msg = ""
        if known is not None and v.any():
            kf = known(t)
            ok = v & (kf > 0)
            msg = " max rel error vs known %.2e" % (np.abs(ref[ok] / kf[ok] - 1).max() if ok.any() else 0.0)
        print("pitch_%s ok: %d samples at %d Hz, %d frames, %d voiced (dio %d)%s" % (name, len(y), sr, F, v.sum(), (f0 > 0).sum(), msg))


if __name__ == "__main__":
    main()
