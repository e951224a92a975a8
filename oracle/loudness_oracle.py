"""ITU-R BS.1770-4 integrated loudness of one channel, in float64, restated from the standard's text (the oracle of
``ev_loudness`` / ``JETSGenerator.measure_loudness``), and the normalisation gain the engine applies.

- K-weighting (Annex 1, section 1.2): a high-shelf pre-filter, then the RLB high-pass.  The standard tables both at 48 kHz; at
  another rate each is the bilinear transform, pre-warped at its corner frequency, of its analog prototype
      shelf      H(s) = (Vh s^2 + Vb (w0 / Q) s + w0^2) / (s^2 + (w0 / Q) s + w0^2)
      high-pass  H(s) = s^2 / (s^2 + (w0 / Q) s + w0^2), numerator taken as the table's b = (1, -2, 1)
  with the corner frequencies, gains and Q that reproduce the 48 kHz table.  The signal is filtered sequentially
  (``scipy.signal.lfilter``, zero initial state).
- Gating (section 2): blocks of 400 ms stepped by 100 ms, only blocks entirely inside the signal; z_j = the block's mean
  square, l_j = -0.691 + 10 log10(z_j); the absolute gate keeps l_j > -70 LKFS, the relative gate sits 10 LU below the
  loudness of the blocks the absolute gate kept, and L is -0.691 + 10 log10(mean z_j over the blocks above both gates).
  L = -inf when no block exists or none passes.
- Gain: g = min(10^((T - L) / 20), 10^(-1/20) / peak), peak = max |x|; 1 where L = -inf.

Shares no code with ``emotivoice_b200.audio``.
"""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view
from scipy.signal import bilinear, lfilter

SHELF_F0, SHELF_GAIN_DB, SHELF_Q, SHELF_VB_EXP = 1681.974450955533, 3.999843853973347, 0.7071752369554196, 0.4996667741545416
HP_F0, HP_Q = 38.13547087602444, 0.5003270373238773
ABS_GATE, REL_GATE, OFFSET = -70.0, -10.0, -0.691
CEILING_DB = -1.0

# BS.1770-4 Annex 1, Tables 1 and 2 (48 kHz)
TABLE_48K = {"shelf_b": (1.53512485958697, -2.69169618940638, 1.19839281085285), "shelf_a": (1.0, -1.69065929318241, 0.73248077421585),
             "hp_b": (1.0, -2.0, 1.0), "hp_a": (1.0, -1.99004745483398, 0.99007225036621)}


def _prewarped(f0, fs):
    return 2.0 * fs * np.tan(np.pi * f0 / fs)


def k_weighting(fs):
    """-> (shelf_b, shelf_a, hp_b, hp_a) float64 arrays of 3 (a[0] = 1) at fs Hz."""
    w0 = _prewarped(SHELF_F0, fs)
    vh = 10.0 ** (SHELF_GAIN_DB / 20.0)
    vb = vh ** SHELF_VB_EXP
    sb, sa = bilinear([vh, vb * w0 / SHELF_Q, w0 * w0], [1.0, w0 / SHELF_Q, w0 * w0], fs)
    w0 = _prewarped(HP_F0, fs)
    _, ha = bilinear([1.0, 0.0, 0.0], [1.0, w0 / HP_Q, w0 * w0], fs)
    return np.asarray(sb, np.float64), np.asarray(sa, np.float64), np.array([1.0, -2.0, 1.0]), np.asarray(ha, np.float64)


def k_filter(x, fs):
    """The K-weighted signal, float64, filtered sequentially from zero state."""
    sb, sa, hb, ha = k_weighting(fs)
    return lfilter(hb, ha, lfilter(sb, sa, np.asarray(x, dtype=np.float64)))


def block_mean_squares(x, fs):
    """z_j of every 400 ms gating block (100 ms step) that lies entirely inside x."""
    y = k_filter(x, fs)
    T, step = 4 * fs // 10, fs // 10
    if len(y) < T:
        return np.zeros(0)
    return sliding_window_view(y * y, T)[::step].mean(axis=1)


def gating(x, fs):
    """-> (L, l, gamma_r): the integrated loudness, every block's loudness l_j and the relative gate (nan when no block passes
    the absolute gate)."""
    z = block_mean_squares(x, fs)
    with np.errstate(divide="ignore"):
        l = OFFSET + 10.0 * np.log10(z)
    keep = l > ABS_GATE
    if not keep.any():
        return -np.inf, l, np.nan
    gamma_r = OFFSET + 10.0 * np.log10(z[keep].mean()) + REL_GATE
    keep &= l > gamma_r
    if not keep.any():
        return -np.inf, l, gamma_r
    return OFFSET + 10.0 * np.log10(z[keep].mean()), l, gamma_r


def integrated_loudness(x, fs):
    return gating(x, fs)[0]


def peak(x):
    return float(np.max(np.abs(np.asarray(x, dtype=np.float64)), initial=0.0))


def gain(L, pk, target):
    """The normalisation gain (float64) of an item with integrated loudness L and sample peak pk to target LUFS."""
    if not np.isfinite(L):
        return 1.0
    return min(10.0 ** ((float(target) - L) / 20.0), 10.0 ** (CEILING_DB / 20.0) / pk)
