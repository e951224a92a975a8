"""TEST INFRASTRUCTURE ONLY -- fp64 numpy restatement of ``pyworld.dio`` and ``pyworld.stonemask`` at pyworld's defaults, the
two calls of the reference's ``feats.Pitch._calculate_pitch`` (models/prompt_tts_modified/feats.py:114-131), and the
reference's glue after them (``_convert_to_continuous_pitch``, the log, ``_average_by_duration``).

NOT CHECKED AGAINST PYWORLD.  Neither pyworld nor WORLD's C++ source is available where this was written.  The restatement
follows the published algorithms (M. Morise et al., "Fast and reliable F0 estimation method based on the period extraction of
vocal fold vibration of singing voice and speech", AES 35th Int. Conf., 2009 -- DIO; and WORLD's StoneMask refinement by
instantaneous frequency) as the author knows WORLD's implementation of them.  Its independent check is accuracy on signals
whose F0 is known (tests/test_pitch.py).  Every point where WORLD's exact behaviour was assumed, and what was chosen:

  DIO (defaults f0_floor 71, f0_ceil 800, channels_in_octave 2, speed 1, allowed_range 0.1)
  D1  Bands: 1 + int(log(800 / 71) / log 2 * 2) = 7, with upper edges b_i = 71 * 2^((i + 1) / 2).
  D2  The analysed signal has y_length = N + 1 samples: the N samples and one zero after them.  The mean is taken over all
      N + 1 and subtracted from all N + 1 (so the last sample is -mean).
  D3  Low-cut: c = round(fs / 50), a (2c + 1)-point Hann window h_j = 0.5 - 0.5 cos(2 pi (j + 1) / (2c + 2)), j = 0..2c,
      normalised by its sequential sum and negated, 1 added at its centre, applied zero-phase.  WORLD applies it and the band
      low-passes by multiplying spectra of one FFT size; at every supported rate that size exceeds the support of the two
      convolutions, so the circular convolution equals the linear one computed here (asserted in ``dio``).  WORLD's copy of
      spectrum bin i into bin fft_size - i - 1 after the product is not reproduced: the inverse real FFT reads bins 0..n/2 only.
  D4  Band low-pass: a (2L + 1)-point Nuttall window, L = round(2 fs / b_i), unnormalised (coefficients 0.355768, 0.487396,
      0.144232, 0.012604), applied causally, then advanced by L + 1 samples: band[i] = sum_k w_k ylc[i + L + 1 - k].
  D5  Events on the band signal v (length N + 1): negative-going zero crossings (v[i] > 0 and v[i + 1] <= 0, edge e = i + 1,
      fine position e - v[e - 1] / (v[e] - v[e - 1])), the same on -v, on d[i] = (-v[i]) - (-v[i + 1]) (peaks, length N) and
      on -d (dips).  Each pair of consecutive events gives an interval fs / (p_{k+1} - p_k) placed at (p_k + p_{k+1}) / 2 / fs.
  D6  A band whose any of the four kinds has at most 2 intervals (fewer than 4 events; digital silence has none) gives no
      candidate: candidate 0, score 100000, at every frame.
  D7  Interpolation at frame times t = i * frame_period / 1000 is MATLAB interp1 via WORLD's histc: linear, extrapolated from
      the first or last pair of intervals outside their range.
  D8  Candidate = mean of the four interpolated values, score = sqrt(sum of squared deviations / 3); rejected (0, 100000) when
      above b_i, below b_i / 2, above f0_ceil or below f0_floor.  The score is then divided by (candidate + 1e-12), and each
      frame takes the band of least score, the lowest band on a tie.
  D9  FixF0Contour with r = int(0.5 + 1000 / frame_period / f0_floor) * 2 + 1 (3 at 16 ms and 12.5 ms frames): when the
      frame count is at most r the contour is all zero.  Step 1 zeroes the first and last r frames and every frame whose
      |f[i] - f[i-1]| / (f[i] + 1e-12) is not below allowed_range.  Step 2 zeroes frames with a zero within +-(r - 1) / 2.
      Steps 3 and 4 extend each voiced section of step 2 forward from its last frame (up to the next section's last frame)
      and backward from its first frame (down to the previous section's first frame, frame 1 at the earliest), taking at each
      frame the band candidate nearest the previous frame's value within allowed_range (relative to that value; the later
      band on a tie) and stopping at the first frame with none.  Sections are taken from step 2's contour, in order.
  STONEMASK
  S1  Frames with F0 <= 40 or F0 > fs / 12 give 0.
  S2  Half window 1.5 / F0, base_time_length = 2 round(1.5 fs / F0) + 1 samples starting at sample
      round((t - round(1.5 fs / F0) / fs) fs + 0.001) - 1, indices clamped to [0, N - 1]; Blackman window
      0.42 + 0.5 cos(2 pi u / W) + 0.08 cos(4 pi u / W), u = (index_raw - 1) / fs - t, W = 3 / F0 + 1 / fs; the difference
      window is -(w[i + 1] - w[i - 1]) / 2 with one-sided ends.  The spectra are of the ORIGINAL samples (no mean removal).
  S3  FFT size 2^(2 + int(log(1.5 fs / F0 + 1) / log 2)).  Only the bins FixF0 reads are formed, as direct DFT sums
      (forward sign), equal to WORLD's FFT bins up to round-off.  A bin past fft_size / 2, which WORLD would read past its
      half spectrum, is taken as the DFT at that index.
  S4  FixF0 at 2 harmonics, rejected (giving the initial F0) when <= 0 or > 2 F0; then at 6 harmonics from that value; bins
      round(f * fft_size / fs * h); instantaneous frequency k fs / n + Im(conj(M) D) / |M|^2 fs / (2 pi) (0 when |M| = 0),
      amplitude-weighted; finally the initial F0 is kept when the result differs from it by more than 20 %.

pyworld's frame count is int(1000 N / fs / frame_period) + 1 in double; with frame_period = 1000 hop / fs that is N // hop + 1
at the supported configurations.  Arithmetic follows WORLD's operation order; scalar transcendental functions are Python's
``math`` (libm) and every sum is sequential, so the results do not depend on numpy's SIMD dispatch.
"""
import math

import numpy as np

F0_FLOOR, F0_CEIL, CHANNELS_IN_OCTAVE, ALLOWED_RANGE = 71.0, 800.0, 2.0, 0.1
CUTOFF = 50.0
MAX_VALUE = 100000.0
SAFE_GUARD = 1e-12
FLOOR_F0_STONEMASK = 40.0
LOG2 = 0.69314718055994529


def matlab_round(x):
    return int(x - 0.5) if x < 0 else int(x + 0.5)


def n_bands():
    return 1 + int(math.log(F0_CEIL / F0_FLOOR) / LOG2 * CHANNELS_IN_OCTAVE)


def boundaries():
    return [F0_FLOOR * math.pow(2.0, (i + 1) / CHANNELS_IN_OCTAVE) for i in range(n_bands())]


def frame_count(n, fs, frame_period):
    return int(1000.0 * n / fs / frame_period) + 1


def voice_range_minimum(frame_period):
    return int(0.5 + 1000.0 / frame_period / F0_FLOOR) * 2 + 1


def lowcut_taps(fs):
    """(c, g): g[j] is the zero-phase tap at offset j - c (D3)."""
    c = matlab_round(fs / CUTOFF)
    n = 2 * c + 1
    w = [0.5 - 0.5 * math.cos(i * 2.0 * math.pi / (n + 1)) for i in range(1, n + 1)]
    s = 0.0
    for v in w:
        s += v
    g = [-v / s for v in w]
    g[c] += 1.0
    return c, np.asarray(g)


def nuttall(n):
    out = []
    for i in range(n):
        tmp = i / (n - 1.0)
        out.append(0.355768 - 0.487396 * math.cos(2.0 * math.pi * tmp) + 0.144232 * math.cos(4.0 * math.pi * tmp)
                   - 0.012604 * math.cos(6.0 * math.pi * tmp))
    return np.asarray(out)


def band_half_lengths(fs):
    return [matlab_round(fs / b * 2.0) for b in boundaries()]


def _fir(xpad, h, count):
    """out[i] = sum_j h[j] xpad[i + j] for i < count, summed over j in ascending order."""
    acc = np.zeros(count)
    for j in range(len(h)):
        acc += h[j] * xpad[j:j + count]
    return acc


def band_signals(x, fs):
    """x (N,) -> (7, N + 1): the band signals of D2-D4."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    m = n + 1
    y = np.zeros(m)
    y[:n] = x
    s = 0.0
    for v in y:                     # sequential: D2
        s += v
    y = y - s / m
    c, g = lowcut_taps(fs)
    halves = band_half_lengths(fs)
    l0 = max(halves)
    # ylc[t] on t in [1 - l0, m + l0]: ylc[t] = sum_j g[j] y[t + c - j]; stored as ylc_ext[t - (1 - l0)]
    cnt = m + 2 * l0
    lo = 1 - l0 - c                  # the first y index read (< 0: zeros before the signal)
    ypad = np.zeros(cnt + 2 * c)
    ypad[-lo:-lo + m] = y
    # sum_j g[j] y[t + c - j] = sum_j g[2c - j] y[t - c + j], summed in ascending j of the second form
    ylc = _fir(ypad, g[::-1], cnt)
    out = np.zeros((len(halves), m))
    for b, L in enumerate(halves):
        w = nuttall(2 * L + 1)
        # band[i] = sum_k w[k] ylc[i + L + 1 - k];  ylc index i + L + 1 - k -> ext index i + L + 1 - k - (1 - l0)
        base = l0 - L                  # ext index of ylc[i + 1 - L] at i = 0 (k = 2L)
        out[b] = _fir(ylc[base:], w[::-1], m)
    return out


def _fine_edges(v):
    """Negative-going zero crossings of v (D5): fine positions."""
    i = np.nonzero((v[:-1] > 0.0) & (v[1:] <= 0.0))[0]
    e = i + 1
    return e.astype(np.float64) - v[e - 1] / (v[e] - v[e - 1])


def events(v):
    """band signal -> [fine positions] of the four kinds: negatives, positives, peaks, dips."""
    neg = _fine_edges(v)
    nv = -v
    pos = _fine_edges(nv)
    d = nv[:-1] - nv[1:]
    peak = _fine_edges(d)
    dip = _fine_edges(-d)
    return [neg, pos, peak, dip]


def intervals(fine, fs):
    """(locations s, values Hz) of consecutive events."""
    return (fine[:-1] + fine[1:]) / 2.0 / fs, fs / (fine[1:] - fine[:-1])


def interp1(x, y, xi):
    k = np.clip(np.searchsorted(x, xi, side="right"), 1, len(x) - 1)
    s = (xi - x[k - 1]) / (x[k] - x[k - 1])
    return y[k - 1] + s * (y[k] - y[k - 1])


def frame_times(F, frame_period):
    return np.arange(F, dtype=np.float64) * frame_period / 1000.0


def band_candidates(v, fs, boundary, t):
    """(candidate, raw score / (candidate + 1e-12), event counts) of one band at frame times t (D6-D8)."""
    ev = events(v)
    F = len(t)
    counts = [len(e) for e in ev]
    if any(len(e) - 1 - 2 <= 0 for e in ev):
        cand = np.zeros(F)
        score = np.full(F, MAX_VALUE)
    else:
        vals = []
        for e in ev:
            loc, val = intervals(e, fs)
            vals.append(interp1(loc, val, t))
        v0, v1, v2, v3 = vals
        cand = (v0 + v1 + v2 + v3) / 4.0
        score = np.sqrt(((v0 - cand) * (v0 - cand) + (v1 - cand) * (v1 - cand) + (v2 - cand) * (v2 - cand)
                         + (v3 - cand) * (v3 - cand)) / 3.0)
        bad = (cand > boundary) | (cand < boundary / 2.0) | (cand > F0_CEIL) | (cand < F0_FLOOR)
        cand = np.where(bad, 0.0, cand)
        score = np.where(bad, MAX_VALUE, score)
    return cand, score / (cand + SAFE_GUARD), counts


def best_contour(cands, scores):
    F = cands.shape[1]
    best = cands[0].copy()
    tmp = scores[0].copy()
    for j in range(1, cands.shape[0]):
        upd = tmp > scores[j]
        tmp = np.where(upd, scores[j], tmp)
        best = np.where(upd, cands[j], best)
    assert best.shape == (F,)
    return best


def _select_best(ref, cands_at):
    best_f0, best_err = 0.0, ALLOWED_RANGE
    for c in cands_at:
        tmp = abs(ref - c) / ref
        if tmp > best_err:
            continue
        best_f0, best_err = c, tmp
    return best_f0


def fix_contour(best, cands, frame_period):
    """FixF0Contour steps 1-4 (D9)."""
    F = len(best)
    r = voice_range_minimum(frame_period)
    out = np.zeros(F)
    if F <= r:
        return out, {"step2": np.zeros(F)}
    base = best.copy()
    base[:r] = 0.0
    base[F - r:] = 0.0
    s1 = np.zeros(F)
    for i in range(r, F):
        s1[i] = base[i] if abs((base[i] - base[i - 1]) / (SAFE_GUARD + base[i])) < ALLOWED_RANGE else 0.0
    s2 = s1.copy()
    ctr = (r - 1) // 2
    for i in range(ctr, F - ctr):
        for j in range(-ctr, ctr + 1):
            if s1[i + j] == 0:
                s2[i] = 0.0
                break
    pos, neg = [], []
    for i in range(1, F):
        if s2[i] == 0 and s2[i - 1] != 0:
            neg.append(i - 1)
        elif s2[i - 1] == 0 and s2[i] != 0:
            pos.append(i)
    s3 = s2.copy()
    for i in range(len(neg)):
        limit = F - 1 if i == len(neg) - 1 else neg[i + 1]
        for j in range(neg[i], limit):
            s3[j + 1] = _select_best(s3[j], cands[:, j + 1])
            if s3[j + 1] == 0:
                break
    s4 = s3.copy()
    for i in range(len(pos) - 1, -1, -1):
        limit = 1 if i == 0 else pos[i - 1]
        for j in range(pos[i], limit, -1):
            s4[j - 1] = _select_best(s4[j], cands[:, j - 1])
            if s4[j - 1] == 0:
                break
    return s4, {"step2": s2}


def dio(x, fs, frame_period, details=False):
    """pyworld.dio(x, fs, frame_period=frame_period) at its other defaults -> (f0, temporal_positions)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    fs = int(fs)
    n = len(x)
    F = frame_count(n, fs, frame_period)
    t = frame_times(F, frame_period)
    c = matlab_round(fs / CUTOFF)
    halves = band_half_lengths(fs)
    fft_size = 2 ** (int(math.log(n + 1 + c * 2 + 1 + 4 * int(1.0 + fs / boundaries()[0] / 2.0)) / LOG2) + 1)
    assert fft_size > n + 1 + 2 * max(halves) + c + 1, "the circular convolution of D3 would alias at fs=%d" % fs
    bands = band_signals(x, fs)
    cands, scores, counts = [], [], []
    for b, bd in enumerate(boundaries()):
        cnd, sc, ct = band_candidates(bands[b], fs, bd, t)
        cands.append(cnd)
        scores.append(sc)
        counts.append(ct)
    cands, scores = np.stack(cands), np.stack(scores)
    best = best_contour(cands, scores)
    f0, st = fix_contour(best, cands, frame_period)
    if details:
        return f0, t, {"candidates": cands, "scores": scores, "best": best, "step2": st["step2"], "counts": np.asarray(counts),
                       "bands": bands}
    return f0, t


_TW = {}


def _twiddles(n):
    tw = _TW.get(n)
    if tw is None:
        a = [2.0 * math.pi * m / n for m in range(n)]
        tw = _TW[n] = (np.asarray([math.cos(v) for v in a]), np.asarray([math.sin(v) for v in a]))
    return tw


def _bin(seg, k, n):
    """DFT bin k (forward sign) of seg zero-padded to n points: (re, im), sequential sums."""
    cos_t, sin_t = _twiddles(n)
    m = (k * np.arange(len(seg))) % n
    re = np.cumsum(seg * cos_t[m])[-1]
    im = -np.cumsum(seg * sin_t[m])[-1]
    return re, im


def _fix_f0(mseg, dseg, fft_size, fs, f0, nh):
    num = den = 0.0
    for i in range(nh):
        index = matlab_round(f0 * fft_size / fs * (i + 1))
        mr, mi = _bin(mseg, index, fft_size)
        dr, di = _bin(dseg, index, fft_size)
        num_i = mr * di - mi * dr
        pw = mr * mr + mi * mi
        inst = 0.0 if pw == 0.0 else index * fs / fft_size + num_i / pw * fs / 2.0 / math.pi
        amp = math.sqrt(pw)
        num += amp * inst
        den += amp * (i + 1.0)
    return num / (den + SAFE_GUARD)


def refine_frame(x, fs, t, f0):
    """GetRefinedF0 (S1-S4) of one frame."""
    n = len(x)
    if f0 <= FLOOR_F0_STONEMASK or f0 > fs / 12.0:
        return 0.0
    hw = 1.5 / f0
    wl = 2.0 * hw + 1.0 / fs
    h = matlab_round(hw * fs)
    btl = h * 2 + 1
    fft_size = int(math.pow(2.0, 2.0 + int(math.log(hw * fs + 1.0) / LOG2)))
    base0 = (-h + 0) / float(fs)
    basic = matlab_round((t + base0) * fs + 0.001)
    raw = basic + np.arange(btl)
    idx = np.clip(raw - 1, 0, n - 1)
    win = np.asarray([0.42 + 0.5 * math.cos(2.0 * math.pi * u / wl) + 0.08 * math.cos(4.0 * math.pi * u / wl)
                      for u in ((r - 1.0) / fs - t for r in raw.tolist())])
    dwin = np.empty(btl)
    dwin[0] = -win[1] / 2.0
    dwin[1:-1] = -(win[2:] - win[:-2]) / 2.0
    dwin[-1] = win[-2] / 2.0
    seg = x[idx]
    mseg, dseg = seg * win, seg * dwin
    tent = _fix_f0(mseg, dseg, fft_size, fs, f0, 2)
    if tent <= 0.0 or tent > f0 * 2:
        mean_f0 = 0.0
    else:
        mean_f0 = _fix_f0(mseg, dseg, fft_size, fs, tent, 6)
    if abs(mean_f0 - f0) > f0 * 0.2:
        mean_f0 = f0
    return mean_f0


def stonemask(x, f0, temporal_positions, fs):
    """pyworld.stonemask(x, f0, temporal_positions, fs)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    return np.asarray([refine_frame(x, int(fs), float(t), float(f)) for t, f in zip(temporal_positions, f0)])


# ---- the reference's glue, restated for the operator checks (the fixtures hold the reference's own outputs) -------------

def continuous(p):
    """feats.py:92-112: held ends and np.interp (scipy interp1d's linear path) between voiced frames."""
    p = np.array(p, dtype=np.float64)
    if (p == 0).all():
        return p
    nz = np.nonzero(p)[0]
    p[:nz[0]] = p[nz[0]]
    p[nz[-1]:] = p[nz[-1]]
    nz = np.nonzero(p)[0]
    return np.interp(np.arange(len(p)).astype(np.float64), nz.astype(np.float64), p[nz])


def log_pitch(p):
    p = np.array(p, dtype=np.float64)
    for i in np.nonzero(p)[0]:
        p[i] = math.log(p[i])
    return p


def average_by_duration(p, d):
    """feats.py:133-147 (its zero mask is a no-op): the mean of each token's frames, 0 for an empty token."""
    d = np.asarray(d, dtype=np.int64)
    cs = np.concatenate([[0], np.cumsum(d)])
    out = []
    for s, e in zip(cs[:-1], cs[1:]):
        a = p[s:e]
        out.append(np.mean(a) if len(a) else 0.0)
    return np.asarray(out, dtype=np.float64)


def pitch(x, fs, hop, use_continuous_pitch=True, use_log_pitch=False):
    """Pitch._calculate_pitch: (raw DIO f0, refined, output)."""
    frame_period = 1000 * hop / fs
    f0, t = dio(x, fs, frame_period)
    ref = stonemask(x, f0, t, fs)
    out = ref.copy()
    if use_continuous_pitch:
        out = continuous(out)
    if use_log_pitch:
        out = log_pitch(out)
    return f0, ref, out
