"""The true-peak limiter of ``format_audio(true_peak=...)`` (``ev_limit``), restated sequentially in float64 numpy.

Per item x of n samples at sr Hz, pre-gain g, ceiling C dBTP:

1. Detector: p[s] = max(|x[s]|, |v| for the interpolated values v between s and s + 1).  The interpolator oversamples by
   R = ceil(192000 / sr) with ``firwin(2 * 10 * R + 1, 1 / R, kaiser 5) * R`` (resample_poly's design).  For an output rate
   below sr the signal is first low-passed with ``firwin(2 * ceil(10 sr / rate) + 1, rate / sr, kaiser 5)`` and all R phases
   are taken.  x is zero outside the item.
2. Required gain r[s] = min(0, C - 20 log10(g p[s])), at least -1000 dB, rounded down to a multiple of Q = 2^-32 dB.
3. Look-ahead and hold: m[s] = min r over [s - M, s + L + M] for s in [-L, n), r = 0 outside the item.
4. Release: the literal recurrence G1[s] = min(m[s], G1[s - 1] + rho), G1[-L - 1] = 0, rho = 60 dB/s per sample rounded to Q.
   ``release_prefix`` is the prefix-minimum form the kernels compute.
5. Attack: G[s] = (sum of G1 over [s - L, s], in index order) / (L + 1).
6. Apply: y[s] = fp32(x[s] * g * 10^(G[s] / 20)).

Two passes with a loudness target T: g1 = 10^((T - L0) / 20), L1 the loudness of the first limited result, g2 = g1 *
10^((T - L1) / 20); each factor is 1 where its loudness is -inf.  Loudness is ``loudness_oracle.integrated_loudness``.

Shares no code with ``emotivoice_b200.audio``.
"""
import math

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view
from scipy.signal import firwin

from oracle import loudness_oracle

DETECT_RATE = 192000
LOOKAHEAD_S = 0.005
RELEASE_DB_PER_S = 60.0
Q = 2.0 ** -32
FLOOR_DB = -1000.0


def oversampling(sr):
    return -(-DETECT_RATE // int(sr))


def lookahead(sr):
    return int(round(LOOKAHEAD_S * sr))


def release(sr):
    return round(RELEASE_DB_PER_S / sr / Q) * Q


def detector_filter(sr, rate):
    """-> (h at the oversampled rate, float64; its half-span c in samples at sr; the phases the detector reads)."""
    R = oversampling(sr)
    h = firwin(2 * 10 * R + 1, 1.0 / R, window=("kaiser", 5.0)) * R
    c = 10
    if rate < sr:
        half = -(-10 * int(sr) // int(rate))
        lp = firwin(2 * half + 1, float(rate) / sr, window=("kaiser", 5.0))
        stuffed = np.zeros(2 * half * R + 1)
        stuffed[::R] = lp
        h = np.convolve(h, stuffed)
        c += half
        return h, c, range(R)
    return h, c, range(1, R)


def hold(sr, rate):
    """M: the larger half-span, in samples at sr, of the detector and of resample_poly's filter for rate / sr."""
    _, c, _ = detector_filter(sr, rate)
    g = math.gcd(int(rate), int(sr))
    up, down = int(rate) // g, int(sr) // g
    return max(c, 0 if up == down else -(-10 * max(up, down) // up))


def detect(x, sr, rate):
    """p[s] of every sample, float64."""
    x = np.asarray(x, np.float64)
    h, c, phases = detector_filter(sr, rate)
    R = oversampling(sr)
    p = np.abs(x)
    for ph in phases:
        hp = h[ph::R]
        y = np.convolve(x, hp)[c:c + len(x)] if len(x) else np.zeros(0)
        p = np.maximum(p, np.abs(y))
    return p


def required(p, g, ceiling):
    with np.errstate(divide="ignore"):
        r = np.minimum(0.0, ceiling - 20.0 * np.log10(g * p))
    r = np.where(p > 0, np.maximum(r, FLOOR_DB), 0.0)
    return np.floor(r / Q) * Q


def hold_min(r, L, M):
    """m[s] for s in [-L, n): index i = s + L."""
    n = len(r)
    padded = np.concatenate([np.zeros(L + M), r, np.zeros(L + M)])
    return sliding_window_view(padded, L + 2 * M + 1)[:n + L].min(axis=1) if n + L else np.zeros(0)


def release_recurrence(m, rho):
    g1 = np.empty(len(m))
    prev = 0.0
    for i in range(len(m)):
        prev = min(m[i], prev + rho)
        g1[i] = prev
    return g1


def release_prefix(m, rho):
    i = np.arange(len(m), dtype=np.float64)
    return np.minimum(0.0, rho * i + np.minimum.accumulate(m - rho * i))


def attack(g1, L):
    """G[s] for s in [0, n) from G1 over [-L, n)."""
    if len(g1) <= L:
        return np.zeros(0)
    return sliding_window_view(g1, L + 1).sum(axis=1) / (L + 1)


def pregain(target, lufs0=None, lufs1=None):
    g = 1.0
    for L in (lufs0, lufs1):
        if L is not None and np.isfinite(L):
            g *= 10.0 ** ((float(target) - float(L)) / 20.0)
    return g


def limit(x, sr, rate, ceiling, g=1.0, fast=False):
    """One pass -> (y float32, envelope G in dB, required r in dB)."""
    x = np.asarray(x, np.float32)
    L, M = lookahead(sr), hold(sr, rate)
    r = required(detect(x, sr, rate), g, ceiling)
    m = hold_min(r, L, M)
    g1 = (release_prefix if fast else release_recurrence)(m, release(sr))
    G = attack(g1, L)
    y = (x.astype(np.float64) * g * 10.0 ** (G / 20.0)).astype(np.float32)
    return y, G, r


def two_pass(x, sr, rate, ceiling, target=None, fast=False):
    """-> (y, G, (L0, L1)): the limited output of format_audio(loudness=target, true_peak=ceiling) at the model's rate."""
    if target is None:
        y, G, _ = limit(x, sr, rate, ceiling, 1.0, fast)
        return y, G, (None, None)
    L0 = loudness_oracle.integrated_loudness(np.asarray(x, np.float64), sr)
    y1, _, _ = limit(x, sr, rate, ceiling, pregain(target, L0), fast)
    L1 = loudness_oracle.integrated_loudness(y1.astype(np.float64), sr)
    y, G, _ = limit(x, sr, rate, ceiling, pregain(target, L0, L1), fast)
    return y, G, (L0, L1)


def true_peak_db(y, rate, edge_s=0.0):
    """True peak (dBTP) of y at ``rate`` Hz: the largest |sample| of y oversampled to at least 192 kHz by resample_poly, fp64.
    ``edge_s``: leave out the first and last edge_s seconds."""
    from scipy.signal import resample_poly
    y = np.asarray(y, np.float64)
    up = -(-DETECT_RATE // int(rate))
    v = np.maximum(np.abs(resample_poly(y, up, 1)), np.repeat(np.abs(y), up)) if len(y) else np.zeros(0)
    e = int(edge_s * rate) * up
    v = v[e:len(v) - e]
    pk = float(np.max(v, initial=0.0))
    return 20.0 * math.log10(pk) if pk > 0 else -math.inf
