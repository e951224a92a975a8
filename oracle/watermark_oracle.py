"""The keyed zero-bit watermark of ``format_audio(watermark=...)`` (``ev_watermark_embed``) and its detector
(``emotivoice_b200.watermark.detect``, ``ev_watermark_detect``), restated from their definitions in float64 numpy.

Everything runs at 16 kHz.

- Transform: the MCLT of frames of N = 1024 samples, hop H = 512, sine window w[n] = sin(pi (n + 1/2) / N).  On the grid
  shifted by tau samples, frame j holds x[(j - 1) H + tau + n], n in [0, N), for j = 0 .. F - 1, F the number of frames that
  start before the end (zero outside [0, len(x))).  C[j, k] = sqrt(2 / H) sum_n w[n] x[..] cos(pi / H (n + 1/2 + H / 2)(k + 1/2)),
  S the same with sin: the MDCT is orthonormal, and the IMDCT of C, overlap-added, gives x back.
- Band: bins 19 .. 217 (about 300 - 3400 Hz).
- Pattern: s(key, r, k) = +1 or -1, r in [0, P), P = 64: -1 when the top bit of mix64(key ^ mix64((r << 10) | k)) is set.
  mix64 is SplitMix64's output function.
- Embed: dC[j, k] = alpha M[j, k] s(key, j mod P, k) in the band, M = sqrt(C^2 + S^2), alpha = 10^(-20 / 20) / sqrt(2);
  y = x + IMDCT(dC) on [0, len(x)).
- Detect: u = C / M in the band (0 where M = 0), b[tau, r, k] = sum of u[tau, j, k] over j = r mod P,
  z(tau, m0) = sum_{r, k} s(key, (r + m0) mod P, k) b[tau, r, k] / sqrt(sum b[tau]^2) (0 when b[tau] is all zero).

Shares no code with ``emotivoice_b200``.  The transforms are direct sums (as matrix products over the frames).
"""
import functools
import math

import numpy as np

N, H, P = 1024, 512, 64
K_LO, K_HI = 19, 218
ALPHA = 10.0 ** (-20.0 / 20.0) / math.sqrt(2.0)
BAND = np.arange(K_LO, K_HI)


def mix64(x):
    """SplitMix64's output function on uint64 values (array in, array out)."""
    z = np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def pattern(key, bins=BAND):
    """(P, len(bins)) float64 of s(key, r, k) = +-1."""
    r = np.arange(P, dtype=np.uint64)[:, None]
    k = np.asarray(bins, dtype=np.uint64)[None, :]
    h = mix64(np.uint64(key) ^ mix64((r << np.uint64(10)) | k))
    return 1.0 - 2.0 * (h >> np.uint64(63)).astype(np.float64)


def window():
    return np.sin(np.pi * (np.arange(N) + 0.5) / N)


def _basis(bins):
    return _basis_of(tuple(int(k) for k in bins))


@functools.lru_cache(maxsize=4)
def _basis_of(bins):
    n = np.arange(N)[:, None] + 0.5 + H / 2
    ph = np.pi / H * n * (np.asarray(bins)[None, :] + 0.5)
    s = math.sqrt(2.0 / H) * window()[:, None]
    return s * np.cos(ph), s * np.sin(ph)


def n_frames(n, tau=0):
    """Frames j >= 0 whose first sample (j - 1) H + tau lies before n."""
    return max(0, (int(n) - int(tau) + 2 * H - 1) // H)


def frames(x, tau=0):
    """(F, N) float64: frame j is x[(j - 1) H + tau + n], zero outside the signal."""
    x = np.asarray(x, dtype=np.float64)
    F = n_frames(len(x), tau)
    pad = np.zeros(F * H + 2 * H)
    lo = H - tau                                   # frame 0 starts at pad[0] = x[tau - H]
    src0 = max(0, -lo)
    m = min(len(x), len(pad) - lo) - src0
    if m > 0:
        pad[lo + src0:lo + src0 + m] = x[src0:src0 + m]
    idx = np.arange(F)[:, None] * H + np.arange(N)[None, :]
    return pad[idx]


def mclt(x, tau=0, bins=BAND):
    """-> (C, S), each (F, len(bins)) float64."""
    cb, sb = _basis(bins)
    fr = frames(x, tau)
    return fr @ cb, fr @ sb


def imdct(C, n, bins=BAND):
    """Overlap-add of the IMDCT of C (F, len(bins)) on the tau = 0 grid, cut to [0, n)."""
    cb, _ = _basis(bins)
    F = C.shape[0]
    out = np.zeros(F * H + 2 * H)
    seg = C @ cb.T
    for j in range(F):
        out[j * H:j * H + N] += seg[j]
    return out[H:H + n]


def embed(x, key, alpha=ALPHA):
    """The marked signal, float64."""
    x = np.asarray(x, dtype=np.float64)
    C, S = mclt(x)
    M = np.hypot(C, S)
    s = pattern(key)
    dC = alpha * M * s[np.arange(C.shape[0]) % P]
    return x + imdct(dC, len(x))


def fold(x, taus=range(H)):
    """b (len(taus), P, band) float64: u = C / M folded modulo P on each grid."""
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros((len(taus), P, len(BAND)))
    for i, tau in enumerate(taus):
        C, S = mclt(x, tau)
        M = np.hypot(C, S)
        u = np.divide(C, M, out=np.zeros_like(C), where=M > 0)
        for j in range(u.shape[0]):
            out[i, j % P] += u[j]
    return out


def z_table(b, key):
    """z (len(taus), P) for each grid of b and each frame phase m0."""
    s = pattern(key)
    A = b @ s.T                                      # A[t, r, q] = sum_k b[t, r, k] s[q, k]
    r = np.arange(P)
    num = np.stack([A[:, r, (r + m0) % P].sum(axis=1) for m0 in range(P)], axis=1)
    den = np.sqrt((b * b).sum(axis=(1, 2)))
    return np.divide(num, den[:, None], out=np.zeros_like(num), where=den[:, None] > 0)


def z_max_keys(b, keys, chunk=100):
    """The largest z over every (tau, m0) of b for each key, by circular correlation along r in the DFT domain."""
    den = np.sqrt((b * b).sum(axis=(1, 2)))
    bf = np.conj(np.fft.rfft(b, axis=1)).transpose(1, 2, 0)          # (f, k, tau)
    out = []
    for i in range(0, len(keys), chunk):
        sf = np.fft.rfft(np.stack([pattern(k) for k in keys[i:i + chunk]]), axis=1).transpose(1, 0, 2)   # (f, key, k)
        z = np.fft.irfft(np.matmul(sf, bf).transpose(1, 2, 0), n=P, axis=2)                             # (key, tau, m0)
        z = np.divide(z, den[None, :, None], out=np.zeros_like(z), where=den[None, :, None] > 0)
        out.append(z.max(axis=(1, 2)))
    return np.concatenate(out)


def detect(x, key, taus=range(H)):
    """The full search -> (largest z, its tau, its m0), the first in (tau, m0) order on ties, and the z table."""
    taus = list(taus)
    z = z_table(fold(x, taus), key)
    i = int(np.argmax(z))
    return float(z.flat[i]), taus[i // P], i % P, z
