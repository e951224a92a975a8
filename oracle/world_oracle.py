"""TEST INFRASTRUCTURE ONLY -- fp64 numpy restatement of ``pyworld.cheaptrick`` (WORLD's CheapTrick spectral envelope) at
pyworld's defaults (q1 = -0.15, f0_floor = 71, fft_size from the rate), and of ``pysptk.sp2mc`` with SPTK's ``freqt``: the
features paper-style mel-cepstral distortion (MCD) is computed from.  ``csrc/world_kernels.cu`` follows it step by step.

NOT CHECKED AGAINST PYWORLD / PYSPTK.  Neither is installed where this was written, nor WORLD's or SPTK's C sources.  The
restatement follows the published algorithm (M. Morise, "CheapTrick, a spectral envelope estimator for high-quality speech
synthesis", Speech Communication 67, 2015) and SPTK's frequency-warping recursion as the author knows their implementations.
Its independent checks are in tests/test_world.py: envelopes recovered from harmonic signals whose envelope is known,
independence of F0 and gain, and the identities of the warping.  Every point where the implementations' exact behaviour was
assumed, and what was chosen:

  CHEAPTRICK (per frame, at time t = f frame_period / 1000 s, item of n samples at fs Hz)
  W1  fft_size = 2^(1 + int(log(3 fs / 71 + 1) / log 2)): 512 at 8 kHz, 1024 at 16 to 24 kHz, 2048 at 44.1 and 48 kHz.
  W2  F0 floor = 3 fs / (fft_size - 3) (GetF0FloorForCheapTrick), not 71: a frame whose F0 is at or below it is analysed at
      500 Hz (kDefaultF0).  Not WORLD's: an F0 above fs / 4 or not finite is analysed at 500 Hz too (WORLD's smoothing would
      read outside the spectrum there).
  W3  Window: h = round(1.5 fs / f0) (MATLAB rounding), 2h + 1 samples at indices clamp(round(t fs + 0.001) + i, 0, n - 1),
      i = -h..h; w_i = 0.5 cos(pi (i / 1.5 / fs) f0) + 0.5, normalised by sqrt(sum w_i^2) (sequential sum).  Then
      x_i w_i minus w_i (sum x_i w_i) / (sum w_i) (sequential sums): the weighted mean removed.
  W4  Power spectrum: |rfft|^2 of the frame zero-padded to fft_size, bins 0..fft_size / 2.
  W5  DC correction (DCCorrection): u = 2 + int(f0 fft_size / fs); bins i < u - 1 gain P(f0 - i fs / fft_size), read by
      interp1Q on the axis f0 - k fs / fft_size, k = 0..u (linear between bins k = int(q) and k + 1, q = (f0 - i fs /
      fft_size) / (fs / fft_size)).
  W6  Linear smoothing of width 2 f0 / 3 (LinearSmoothing): b = int(width fft_size / fs) + 1 bins mirrored on each side
      (bins b..1 before bin 0, bins fft_size / 2 .. fft_size / 2 - b after bin fft_size / 2 - 1), m = that times
      fs / fft_size; WORLD reads its running sum S by interp1Q on an axis starting at -(b - 0.5) fs / fft_size, at
      x = i fs / fft_size - width / 2 (low) and at x + width (high), and takes (high - low) / width.  With q = (x - origin) /
      (fs / fft_size), l = int(q), f = q - l for the low read and h, g likewise for the high one, high - low is in exact
      arithmetic m[l+1] (1 - f) + m[l+2] + ... + m[h] + m[h+1] g (m past the end 0), and that local sum (ascending) is what
      is computed.  Not WORLD's rounding: WORLD's difference of two sums of the whole spectrum loses every digit below
      ulp(S) in quiet bands (there it can even be negative, by an ulp), where the local sum of non-negative terms keeps them
      and is never negative.  The two differ by a few ulp(S) / width, the size of WORLD's own |randn| eps noise (W7).
  W7  Noise: WORLD adds randn * 1e-12 to the windowed samples and |randn| * eps to the smoothed power, from a generator whose
      state runs across frames.  Both are replaced by a deterministic floor: eps = 2.220446049250313e-16 is added to every
      smoothed power bin.  A frame's envelope then depends on its own samples only, and digital silence gives log(eps).
  W8  Cepstrum: log of the floored power, extended evenly to fft_size points, its rfft (real part); times the smoothing lifter
      sin(pi f0 q) / (pi f0 q) (1 at q = 0) and the compensation lifter (1 - 2 q1) + 2 q1 cos(2 pi f0 q), q = k / fs, and
      divided by fft_size; the inverse real FFT of that (imaginary parts 0), bins 0..fft_size / 2, then exp.
  W9  Frames: F_b = int(1000 n / fs / frame_period) + 1 (pitch_track's count); frames at or past F_b are 0.

  SP2MC (pysptk.sp2mc(sp, order, alpha))
  W10 c = irfft(log sp) (fft_size = 2 (bins - 1) coefficients), c[0] /= 2, then freqt(c, order, alpha).
  W11 freqt is SPTK's recursion over all fft_size coefficients of c, the mirror half c[fft_size / 2 + 1 ..] included, as
      pysptk passes them: for c[m1], c[m1 - 1], ..., c[0] (m1 = fft_size - 1): d = g; g0 = c[i] + a d0; g1 = (1 - a^2) d0 +
      a d1; gj = d(j-1) + a (dj - g(j-1)), j = 2..order.  The result is linear in log sp: ``sp2mc_table`` is its matrix.

Transcendental functions are numpy's (libm-accurate in fp64); the FFTs are numpy's pocketfft.  Sums the definition fixes
(window energy, weighted mean, the smoothing's local sums) are sequential."""
import math

import numpy as np

Q1 = -0.15
F0_FLOOR = 71.0
DEFAULT_F0 = 500.0
EPS = 2.220446049250313e-16


def fft_size(fs):
    """W1."""
    return 2 ** (1 + int(math.log(3.0 * fs / F0_FLOOR + 1.0) / math.log(2.0)))


def f0_floor(fs, n_fft):
    """W2."""
    return 3.0 * fs / (n_fft - 3.0)


def matlab_round(x):
    return int(x - 0.5) if x < 0 else int(x + 0.5)


def frame_count(n, fs, frame_period):
    return int(1000.0 * n / fs / frame_period) + 1


def analysis_f0(f0, fs, n_fft):
    """W2: the F0 a frame is analysed at."""
    f0 = float(f0)
    if not (f0 > f0_floor(fs, n_fft) and f0 <= fs / 4.0):
        return DEFAULT_F0
    return f0


def _seq_sum(v):
    return float(np.cumsum(v)[-1])


def interp1q(x0, dx, y, xi):
    """WORLD's interp1Q: y sampled at x0 + k dx, read at xi (linear; delta past the last sample 0)."""
    y = np.asarray(y, np.float64)
    dy = np.append(y[1:] - y[:-1], 0.0)
    q = (np.asarray(xi, np.float64) - x0) / dx
    base = q.astype(np.int64)                    # truncation, as static_cast<int>
    return y[base] + dy[base] * (q - base)


def windowed(x, n, fs, f0, t, n_fft):
    """W3: the frame, zero-padded to n_fft."""
    h = matlab_round(1.5 * fs / f0)
    base = np.arange(-h, h + 1)
    origin = matlab_round(t * fs + 0.001)
    idx = np.clip(origin + base, 0, n - 1)
    w = 0.5 * np.cos(math.pi * (base / 1.5 / fs) * f0) + 0.5
    w = w / math.sqrt(_seq_sum(w * w))
    seg = np.asarray(x, np.float64)[idx] * w
    seg = seg - w * (_seq_sum(seg) / _seq_sum(w))
    out = np.zeros(n_fft)
    out[:2 * h + 1] = seg
    return out


def dc_correction(p, f0, fs, n_fft):
    """W5."""
    u = 2 + int(f0 * n_fft / fs)
    axis = np.arange(u, dtype=np.float64) * fs / n_fft
    rep = interp1q(f0, -float(fs) / n_fft, p[:u + 1], axis[:u - 1])
    out = p.copy()
    out[:u - 1] = p[:u - 1] + rep
    return out


def linear_smoothing(p, width, fs, n_fft):
    """W6."""
    half = n_fft // 2
    b = int(width * n_fft / fs) + 1
    mirror = np.concatenate([p[b:0:-1], p[:half], p[half:half - b - 1:-1]])
    assert mirror.size == half + 2 * b + 1
    m = np.append(mirror * fs / n_fft, 0.0)                                # m[ml] = 0: interp1Q's last delta
    origin = -(b - 0.5) * fs / n_fft
    df = float(fs) / n_fft
    axis = np.arange(half + 1, dtype=np.float64) / n_fft * fs - width / 2.0
    ql, qh = (axis - origin) / df, ((axis + width) - origin) / df
    lo, hi = ql.astype(np.int64), qh.astype(np.int64)                     # truncation, as static_cast<int>
    fl, fh = ql - lo, qh - hi
    same = hi == lo
    acc = np.where(same, m[lo + 1] * (fh - fl), m[lo + 1] * (1.0 - fl))
    for o in range(2, int((hi - lo).max()) + 1):                           # m[l+2] .. m[h], ascending, per bin
        j = lo + o
        acc = acc + np.where(j <= hi, m[np.minimum(j, m.size - 1)], 0.0)
    acc = acc + np.where(same, 0.0, m[np.minimum(hi + 1, m.size - 1)] * fh)
    return acc / width


def envelope_frame(x, n, fs, f0, t, n_fft, log=False):
    """One frame of CheapTrick -> (n_fft // 2 + 1,) power envelope (or its log before the exp, with log=True)."""
    f0 = analysis_f0(f0, fs, n_fft)
    half = n_fft // 2
    frame = windowed(x, n, fs, f0, t, n_fft)
    spec = np.fft.rfft(frame)
    p = spec.real * spec.real + spec.imag * spec.imag
    p = dc_correction(p, f0, fs, n_fft)
    p = linear_smoothing(p, f0 * 2.0 / 3.0, fs, n_fft)
    p = p + EPS                                                            # W7
    lg = np.log(p)
    full = np.concatenate([lg, lg[half - 1:0:-1]])
    cep = np.fft.fft(full).real                                            # W8
    q = np.arange(half + 1, dtype=np.float64) / fs
    with np.errstate(invalid="ignore", divide="ignore"):
        smooth = np.where(q == 0, 1.0, np.sin(math.pi * f0 * q) / (math.pi * f0 * q))
    comp = (1.0 - 2.0 * Q1) + 2.0 * Q1 * np.cos(2.0 * math.pi * q * f0)
    lifted = cep[:half + 1] * smooth * comp / n_fft
    out = np.fft.irfft(lifted, n_fft) * n_fft                             # FFTW's unnormalised c2r
    out = out[:half + 1]
    return out if log else np.exp(out)


def cheaptrick(x, fs, f0, frame_period, n=None, log=False):
    """An item's envelopes: x its samples (n of them, default len(x)), f0 (F,) per frame -> (F, fft_size // 2 + 1), frames
    at or past F_b zero (W9)."""
    n = len(x) if n is None else int(n)
    n_fft = fft_size(fs)
    F = len(f0)
    Fb = min(frame_count(n, fs, frame_period), F)
    out = np.zeros((F, n_fft // 2 + 1))
    for f in range(Fb):
        out[f] = envelope_frame(x, n, fs, f0[f], f * frame_period / 1000.0, n_fft, log)
    return out


def freqt(c, order, alpha):
    """W11: SPTK freqt of c (any length) -> order + 1 coefficients."""
    c = np.asarray(c, np.float64)
    b = 1.0 - alpha * alpha
    g = np.zeros(order + 1)
    for i in range(len(c) - 1, -1, -1):
        d = g.copy()
        g[0] = c[i] + alpha * d[0]
        if order >= 1:
            g[1] = b * d[0] + alpha * d[1]
        for j in range(2, order + 1):
            g[j] = d[j - 1] + alpha * (d[j] - g[j - 1])
    return g


def sp2mc(sp, order, alpha):
    """W10: (bins,) power envelope -> (order + 1,) mel-cepstrum."""
    sp = np.asarray(sp, np.float64)
    c = np.fft.irfft(np.log(sp))
    c[0] /= 2.0
    return freqt(c, order, alpha)


def warped_frequency(omega, alpha):
    """The all-pass (first-order) frequency warping of freqt: omega -> omega + 2 atan(alpha sin / (1 - alpha cos))."""
    return omega + 2.0 * np.arctan(alpha * np.sin(omega) / (1.0 - alpha * np.cos(omega)))
