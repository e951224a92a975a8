"""What the recording-analysis API accepts, sorted into the classes that change a kernel's code path, and the representative
cases tests/test_analysis_kernels_gpu.py checks the kernels at.

* stft_feats_kernel (``TacotronSTFT``, ``mel_spectrogram_torch``, ``Energy``): hop 1 .. 1024 (the tile of 32 frames stages
  hop * 31 + 1024 samples; mel_spectrogram_torch pads (1024 - hop) // 2, which floors at odd hops and is 0 at 1024), 1 .. 128
  mel bands (each lane takes bands j, j + 32, ..: one to four rounds), the band table of the basis (empty bands, single-bin
  bands, fmin > 0, fmax = sr / 2) and the sample rate the basis is built for;
* ev_pitch: integer rates 8000 .. 48000 (the low-cut length 2 round(fs / 50) + 1, StoneMask's fs / 12 gate, which binds below
  9600 Hz only), hops 16 .. 4096 (FixF0Contour's width r) and the lengths where pyworld's frame count is not n // hop + 1;
* ev_world_envelope and ev_sp2mc: the hop edges, the output rows of ``table_products`` (one warp per row, 8 rows a round, at
  most 256), the bins of the envelope (3 .. 1025) and the all-pass constant alpha (|alpha| < 1).

``*_CASES`` list the representatives with why each is there; ``*_classes()`` name the sets that must each hold one, and
``uncovered`` names the classes a list of cases leaves empty.
"""
import functools

from emotivoice_b200 import feats

# ---- STFT --------------------------------------------------------------------------------------------------------------------
TILE = 32                               # frames per stft_feats_kernel CTA
WARPS = 8
STFT_HOPS = range(1, feats.N_FFT + 1)
STFT_MELS = range(1, 129)
STFT_RATES = (8000, 16000, 22050, 24000, 44100, 48000)
STFT_RANGES = ((0.0, 8000.0), (0.0, None), (80.0, 7600.0))   # (fmin, fmax): the recipes' 0-8 kHz, up to sr / 2, fmin > 0
SMEM_MAX = 227 * 1024


def stft_smem(hop, n_mels):
    """stft_feats_kernel's dynamic shared memory (feats_smem_bytes)."""
    return 4 * (2 * 1024 + 1024 + 2 * WARPS * (512 + 64) + WARPS * 516 + (n_mels + 1) * TILE + hop * (TILE - 1) + 1024)


def mt_pad(hop):
    """mel_spectrogram_torch's reflect padding."""
    return (feats.N_FFT - hop) // 2


def pad_of(variant, hop):
    return mt_pad(hop) if variant == "mt" else feats.N_FFT // 2


@functools.lru_cache(maxsize=None)
def band_kinds(sr, n_mels, fmin, fmax):
    """-> (empty bands, single-bin bands) of feats.band_table(mel_filterbank(...)) at the FFT size 1024."""
    bt, _ = feats.band_table(feats.mel_filterbank(sr, feats.N_FFT, n_mels, fmin, fmax))
    return int((bt[:, 1] == 0).sum()), int((bt[:, 1] == 1).sum())


# variant, sample rate, mel bands (None: energy only), fmin, fmax, hop: why it is here
STFT_CASES = [
    (("taco", 22050, 80, 0.0, 8000.0, 256), "TacotronSTFT() at the reference's defaults: 3 rounds of bands"),
    (("energy", 24000, None, None, None, 300), "Energy(sr=24000, n_fft=1024, hop_length=300): Pitch's and Energy's hop"),
    (("mt", 8000, 80, 0.0, 8000.0, 1), "lowest hop; 17 empty bands (fmax = sr / 2 at 8 kHz); odd hop, padding 511"),
    (("taco", 16000, 1, 0.0, 8000.0, 2), "one band; smallest even hop"),
    (("mt", 44100, 128, 0.0, 8000.0, 255), "four rounds of bands; 51 single-bin bands; odd hop"),
    (("taco", 48000, 128, 0.0, 8000.0, 257), "one empty and 55 single-bin bands"),
    (("mt", 16000, 32, 80.0, 7600.0, 511), "one full round of bands; fmin > 0; padding 256 (511 / 2 floored)"),
    (("taco", 24000, 33, 0.0, None, 1023), "one band past a full round; fmax = sr / 2; largest odd hop"),
    (("mt", 48000, 128, 0.0, 8000.0, 1024), "highest hop: most shared memory, mel_spectrogram_torch pads 0"),
    (("energy", 8000, None, None, None, 1024), "energy alone at the highest hop"),
]


def stft_classes():
    """name -> (field, set of values): a case is in the class when its field is in the set."""
    hops = set(STFT_HOPS)
    c = {
        "hop: lowest (1)": ("hop", {1}),
        "hop: smallest even (2)": ("hop", {2}),
        "hop: odd, mel_spectrogram_torch's padding floors": ("hop", {h for h in hops if h % 2}),
        "hop: even": ("hop", {h for h in hops if h % 2 == 0}),
        "hop: either side of the default 256": ("hop", {255, 257}),
        "hop: TacotronSTFT's and mel_spectrogram_torch's 256": ("hop", {256}),
        "hop: Energy's and Pitch's 300": ("hop", {300}),
        "hop: half a frame less one (511)": ("hop", {511}),
        "hop: largest odd (1023)": ("hop", {1023}),
        "hop: highest (1024), mel_spectrogram_torch pads 0": ("hop", {h for h in hops if mt_pad(h) == 0}),
        "variant TacotronSTFT": ("variant", {"taco"}),
        "variant mel_spectrogram_torch": ("variant", {"mt"}),
        "variant Energy": ("variant", {"energy"}),
    }
    for r in range(1, 5):
        c["bands: %d round(s) of the band loop" % r] = ("n_mels", {m for m in STFT_MELS if (m + 31) // 32 == r})
    c["bands: one"] = ("n_mels", {1})
    c["bands: a full round (32)"] = ("n_mels", {32})
    c["bands: one past a full round (33)"] = ("n_mels", {33})
    c["bands: TacotronSTFT's 80"] = ("n_mels", {80})
    c["bands: most (128)"] = ("n_mels", {max(STFT_MELS)})
    for sr in STFT_RATES:
        c["rate %d Hz" % sr] = ("sr", {sr})
    tables = [(sr, m, lo, hi) for sr in STFT_RATES for m in (1, 32, 33, 80, 128) for lo, hi in STFT_RANGES]
    c["band table with an empty band"] = ("table", {t for t in tables if band_kinds(*t)[0] > 0})
    c["band table with a single-bin band"] = ("table", {t for t in tables if band_kinds(*t)[1] > 0})
    c["band table with fmin > 0"] = ("table", {t for t in tables if t[2] > 0})
    c["band table up to sr / 2"] = ("table", {t for t in tables if t[3] is None or t[3] == t[0] / 2})
    most = max(stft_smem(h, m) for h in STFT_HOPS for m in STFT_MELS)
    c["most shared memory"] = ("smem", {most})
    return c


def stft_fields(case):
    variant, sr, n_mels, fmin, fmax, hop = case
    return {"variant": variant, "sr": sr, "n_mels": n_mels, "hop": hop,
            "table": None if n_mels is None else (sr, n_mels, fmin, fmax), "smem": stft_smem(hop, n_mels or 0)}


# ---- pitch -------------------------------------------------------------------------------------------------------------------
PITCH_RATES = range(feats.PITCH_SR_RANGE[0], feats.PITCH_SR_RANGE[1] + 1)
PITCH_HOPS = range(feats.PITCH_HOP_RANGE[0], feats.PITCH_HOP_RANGE[1] + 1)


def lowcut_half(fs):
    """DIO's low-cut half length c = round(fs / 50) (MATLAB rounding)."""
    return int(fs / 50.0 + 0.5)


def band_halves(fs):
    """DIO's seven band half-lengths round(2 fs / b_i), b_i = 71 * 2^((i + 1) / 2)."""
    return [int(fs / (71.0 * 2.0 ** ((i + 1) / 2.0)) * 2.0 + 0.5) for i in range(7)]


def fix_width(fs, hop):
    """FixF0Contour's r = int(0.5 + 1000 / frame_period / 71) * 2 + 1."""
    return int(0.5 + 1000.0 / feats.pitch_frame_period(fs, hop) / 71.0) * 2 + 1


# rate: (hop, why it is here)
PITCH_RATE_CASES = {
    8000: (80, "lowest rate; StoneMask's fs / 12 = 666.7 Hz gate binds below DIO's 800 Hz ceiling"),
    11025: (128, "fs / 50 = 220.5: the low-cut length sits on MATLAB round's half"),
    16000: (256, "the project's rate"),
    22050: (256, "TacotronSTFT's rate; pyworld's frame count differs from n // hop + 1"),
    24000: (300, "Pitch()'s defaults"),
    32000: (320, "a rate between the tested ones: c = 640"),
    44100: (441, "CD rate"),
    48000: (480, "highest rate: c = 960, l0 = 956"),
}
PITCH_HOP_EDGES = [(8000, 16), (8000, 4096), (48000, 16), (48000, 4096)]
FRAME_COUNT_LENGTHS = {(22050, 256): [3328, 6656, 13312]}


def pitch_configs():
    """The (fs, hop) pairs the pitch cases run at."""
    return sorted({(fs, h) for fs, (h, _) in PITCH_RATE_CASES.items()} | set(PITCH_HOP_EDGES))


def pitch_classes():
    """name -> set of (fs, hop) or of rates; each must hold a representative."""
    rates = set(PITCH_RATES)
    lo, hi = min(PITCH_RATES), max(PITCH_RATES)
    hlo, hhi = min(PITCH_HOPS), max(PITCH_HOPS)
    c = {
        "rate: lowest": ("fs", {lo}),
        "rate: highest": ("fs", {hi}),
        "rate: StoneMask's fs / 12 gate below DIO's ceiling (fs < 9600)": ("fs", {r for r in rates if r / 12.0 < 800.0}),
        "rate: StoneMask's gate above DIO's ceiling": ("fs", {r for r in rates if r / 12.0 >= 800.0}),
        "rate: fs / 50 on MATLAB round's half": ("fs", {r for r in rates if r % 50 == 25}),
        "rate: fs / 50 whole": ("fs", {r for r in rates if r % 50 == 0}),
        "config: lowest hop at the lowest rate": ("config", {(lo, hlo)}),
        "config: highest hop at the lowest rate (r = 1: a median of width 0)": ("config", {(lo, hhi)}),
        "config: lowest hop at the highest rate (largest r)": ("config", {(hi, hlo)}),
        "config: highest hop at the highest rate": ("config", {(hi, hhi)}),
        "config: Pitch()'s defaults (24000, 300)": ("config", {(24000, 300)}),
    }
    for r in (16000, 22050, 32000, 44100):
        c["rate: %d Hz" % r] = ("fs", {r})
    mismatch = set()
    for fs, hop in pitch_configs():
        mismatch |= {(fs, hop, n) for n in range(feats.pitch_min_samples(fs), 2 * fs)
                     if feats.pitch_frames(n, fs, hop) != n // hop + 1}
    c["length: pyworld's frame count is not n // hop + 1"] = ("length", mismatch)
    return c


def pitch_fields():
    """The fields the pitch cases cover, as sets."""
    cfg = pitch_configs()
    return {"fs": {fs for fs, _ in cfg}, "config": set(cfg),
            "length": {(fs, hop, n) for (fs, hop), ns in FRAME_COUNT_LENGTHS.items() for n in ns}}


# ---- WORLD envelope and mel-cepstrum -----------------------------------------------------------------------------------------
WORLD_ROWS = range(1, feats.SP2MC_MAX_ORDER + 2)
WORLD_BINS = [2 ** k + 1 for k in range(1, 11)]           # fft_size // 2 + 1, fft_size 4 .. 2048
WORLD_HOP_EDGES = [(8000, 16), (48000, 16), (8000, 4096), (48000, 4096)]
WORLD_ROW_CASES = {1: "one row", 8: "one full round of 8 warps", 9: "one past a round", 25: "c0..c24, the recipes' order 24",
                   33: "a fifth round", 256: "most rows: order 255"}
WORLD_BIN_CASES = {3: "fewest bins (fft_size 4), fewer than a warp's lanes", 257: "8 kHz envelope (fft_size 512)",
                   513: "16 to 24 kHz envelope", 1025: "44.1 and 48 kHz envelope: most bins"}
WORLD_ALPHAS = (0.42, -0.99, 0.99)


def world_classes():
    rounds = lambda k: (k + 7) // 8                                   # noqa: E731
    env_bins = {feats.world_fft_size(fs) // 2 + 1 for fs in PITCH_RATES}
    c = {
        "rows: one": ("rows", {1}),
        "rows: one full round": ("rows", {8}),
        "rows: one past a round": ("rows", {9}),
        "rows: ending in the fourth round": ("rows", {k for k in WORLD_ROWS if rounds(k) == 4}),
        "rows: a fifth round or later": ("rows", {k for k in WORLD_ROWS if rounds(k) >= 5}),
        "rows: most (order 255)": ("rows", {max(WORLD_ROWS)}),
        "bins: fewest": ("bins", {min(WORLD_BINS)}),
        "bins: most": ("bins", {max(WORLD_BINS)}),
        "hop edge: lowest hop": ("hop", {min(PITCH_HOPS)}),
        "hop edge: highest hop": ("hop", {max(PITCH_HOPS)}),
        "alpha: near -1": ("alpha", {a for a in WORLD_ALPHAS if a <= -0.9}),
        "alpha: near +1": ("alpha", {a for a in WORLD_ALPHAS if a >= 0.9}),
    }
    for b in sorted(env_bins):
        c["bins: an envelope's %d" % b] = ("bins", {b})
    return c


def world_fields():
    return {"rows": set(WORLD_ROW_CASES), "bins": set(WORLD_BIN_CASES), "hop": {h for _, h in WORLD_HOP_EDGES},
            "alpha": set(WORLD_ALPHAS)}


# ---- coverage ----------------------------------------------------------------------------------------------------------------
def uncovered(classes, covered):
    """The names of ``classes`` (name -> (field, members)) that ``covered`` (field -> set of values) leaves empty."""
    return sorted(name for name, (field, members) in classes.items() if not members & covered.get(field, set()))


def stft_covered(cases):
    out = {}
    for case in cases:
        for k, v in stft_fields(case).items():
            if v is not None:
                out.setdefault(k, set()).add(v)
    return out
