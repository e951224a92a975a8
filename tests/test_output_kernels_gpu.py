"""The output chain's kernels against their fp64 oracles at every representative output rate (tests/output_plans.py), with
lengths on the kernels' tile and loop edges:

* ev_format_audio (audio_out_kernel) against resample_poly in fp64 at all twelve plans, in float32, PCM16, mu-law and A-law,
  |y - y64| <= 2^-16 m as in test_audio_format_gpu (m the sum of |tap * sample| entering the output), PCM16 exact away from
  rounding ties, G.711 equal to tests/golden/g711.npz.  A batch of 64 NaN-padded items: outputs of 1, 255, 256, 257, 512 and
  513 samples (the input lengths on either side of each where up > down makes them unreachable), one item of more 256-output
  tiles than the CTAs per item, so the grid-stride loop turns, and random lengths.  Each item equals its batch-1 call and its
  place in the reversed list bit for bit, nothing is written past the packed outputs, and with a gain each output is
  fp32(acc) * g.
* ev_limit (lim_*) against limiter_oracle.limit at the detector bank of every representative rate (the rates from 16 kHz up
  share one bank and hold), REL = 1e-5 on samples and 1e-4 dB on the envelope as in test_limiter_gpu, n in {1, L - 1, L, L + 1}
  and n + L in {1023, 1024, 1025, 2047, 2048, 2049} around the 1024-index tiles, and a long item that limits in every tile.
* ev_loudness (loud_*) against loudness_oracle at 8, 16 and 48 kHz within 1e-3 LU (no block within 0.01 LU of a gate), peak
  exact: sub-block counts 31, 32, 33 (a warp's 32), 128, 129 (a CTA's 128) and 257 (the gate kernel's 256-thread loop), whole
  and with one extra sample that holds the peak, and block counts 255, 256, 257; a full-scale 1 kHz sine reads -3.01 LUFS.
* ev_watermark_embed (wm_embed_kernel) against watermark_oracle.embed within EMBED_TOL of the peak around the 7-hop (3584-sample)
  tiles and over 40,000 samples (79 frames, so the 64-frame pattern wraps), nothing written past any item.
* ev_watermark_detect (wm_detect_kernel, wm_pick_kernel) against watermark_oracle.detect's full search on marked noise of
  40,000 samples (80 frames per offset, so the fold wraps), 513 and 300 (shorter than a hop): per-offset best z within Z_TOL,
  the best phase wherever the top two are more than 2 Z_TOL apart.  Z_TOL is a measured figure, not a derived bound, and it
  does not hold for every signal: on a marked speech-like item of 40,000 samples the per-offset error reached 2.05e-3.  Each
  cell adds u = C / M, and where M is a small fraction of its frame's energy (between harmonics, high in the band) the FFT's
  fp32 rounding is a large fraction of M.  Evidence that this is conditioning and not the fold: noise of the same length
  stays at 3e-6, and the detector restated in fp32 numpy (scipy's single-precision FFT) gives 7e-4 on the same speech-like
  item.  That item is run and its error printed, not asserted.
* ev_flac_encode (flac_*) against flac_oracle byte for byte at every representative rate, so frame-header rate codes 12, 13,
  14 and 0 all run, directly and through fetch_audio; and one item of 2049 * 4096 + 257 samples: 3-byte frame numbers and a
  257-sample last block.

Worst error against each bound, measured on an H100 80GB HBM3 (132 SMs, 700 W power limit):
    audio_out_kernel  err / m  3.97e-7 (192 kHz; 2.4e-7 .. 4.0e-7 over the plans, 0 for the copy), bound 2^-16 = 1.53e-5
    lim_*             sample rel 4.72e-7 (bound 1e-5), envelope 3.75e-6 dB (bound 1e-4), both at the 8 kHz bank
    loud_*            |L - L64| 3.44e-6 LU at 48 kHz (1.55e-6 at 8 kHz, 3.16e-6 at 16 kHz), bound 1e-3; peaks exact
    wm_embed_kernel   |y - y64| / peak 6.18e-8, bound EMBED_TOL = 1e-6
    wm_detect_kernel  per-offset |z - z64| 3.07e-6 on noise, bound Z_TOL = 1e-3
    flac_*            every image byte-identical at all twelve rates and on the 8,392,961-sample item
The whole file took 77 s there.
"""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import output_plans as P
from audio_cases import SR, abi_limit, out_dict, padded_batch
from emotivoice_b200 import _abi, audio
from emotivoice_b200 import frontdoor as fd
from oracle import flac_oracle as F
from oracle import limiter_oracle as LO
from oracle import loudness_oracle as LU
from oracle import watermark_oracle as W
from test_audio_format_gpu import TAU, _check_float32, _check_pcm16, _g711, _reference
from test_flac_gpu import abi_flac
from test_limiter_gpu import ENV_DB, REL, _compare
from test_loudness_gpu import DL
from test_watermark import speech_like
from test_watermark_gpu import EMBED_TOL, KEY, Z_TOL, abi_detect, abi_embed

pytestmark = pytest.mark.gpu
RATES = sorted(P.REPRESENTATIVE_RATES)
AO_CTAS_PER_SM = 8              # audio_out_kernel's grid: 8 CTAs per SM shared among the listed items
BATCH = 64
LONG_TILES = 40


def _worst(kernel, value):
    print("worst %s: %.3g" % (kernel, value))


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


# ---- ev_format_audio ------------------------------------------------------------------------------------------------

ENC_DTYPES = {"float32": np.float32, "pcm16": np.int16, "mulaw": np.uint8, "alaw": np.uint8}
GUARD, FILL = 256, 0xA5


def abi_format(lib, dev, w, lens, up, down, enc, items=None, gain=None):
    """ev_format_audio straight through the ABI -> one host array per listed item; asserts nothing is written past them."""
    wt = torch.from_numpy(w).to(dev)
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    listed = list(range(len(lens))) if items is None else list(items)
    it = None if items is None else torch.tensor(listed, dtype=torch.int64, device=dev)
    offs = audio.packed_offsets(lens, listed, up, down)
    off = torch.from_numpy(offs[:-1].copy()).to(dev)
    bank = None if (up, down) == (1, 1) else torch.from_numpy(audio.polyphase_bank(up, down)).to(dev)
    g = None if gain is None else torch.from_numpy(np.asarray(gain, np.float32)).to(dev)
    size = np.dtype(ENC_DTYPES[enc]).itemsize
    dst = torch.full(((int(offs[-1]) + GUARD) * size,), FILL, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_format_audio(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None if it is None else it.data_ptr(), len(listed),
                                   off.data_ptr(), None if bank is None else bank.data_ptr(), up, down,
                                   0 if bank is None else bank.shape[1], audio.ENCODINGS[enc], dst.data_ptr(),
                                   None if g is None else g.data_ptr(), _stream(dev)))
    raw = dst.cpu().numpy()
    assert np.all(raw[int(offs[-1]) * size:] == FILL), (up, down, enc)
    y = raw[:int(offs[-1]) * size].view(ENC_DTYPES[enc])
    return [y[offs[k]:offs[k + 1]] for k in range(len(listed))]


def _bracket(m, up, down):
    """Input lengths on either side of m outputs: the largest n with at most m, the smallest with at least m."""
    return {n for n in ((m * down) // up, ((m - 1) * down) // up + 1) if n >= 1}


def format_lengths(up, down, seed):
    lens = set()
    for m in (1, 255, 256, 257, 512, 513):
        lens |= _bracket(m, up, down)
    lens = sorted(lens)
    lens.append(max(_bracket(LONG_TILES * 256 + 77, up, down)))
    rng = np.random.default_rng(seed)
    lens += [int(n) for n in rng.integers(1, 3000, BATCH - len(lens))]
    return lens


def _noise_batch(lens, seed):
    rng = np.random.default_rng(seed)
    return padded_batch([np.tanh(rng.standard_normal(n) * 0.8).astype(np.float32) for n in lens])[0]


@pytest.mark.parametrize("rate", RATES)
def test_format_audio_matches_resample_poly_at_every_plan(lib, dev, rate):
    _, up, down = audio.plan(rate, "pcm16", SR)
    lens = format_lengths(up, down, rate)
    w = _noise_batch(lens, rate)
    long_tiles = -(-audio.resampled_length(max(lens), up, down) // 256)
    per_item = -(-AO_CTAS_PER_SM * torch.cuda.get_device_properties(dev).multi_processor_count // BATCH)
    assert long_tiles > per_item, (long_tiles, per_item)
    got = {enc: abi_format(lib, dev, w, lens, up, down, enc) for enc in ENC_DTYPES}
    tables = _g711()
    worst = 0.0
    for b, n in enumerate(lens):
        x = w[b, 0, :n]
        assert len(got["float32"][b]) == audio.resampled_length(n, up, down)
        y64, m = _reference(x, up, down)
        _check_float32(got["float32"][b], y64, m)
        worst = max(worst, float(np.max(np.abs(got["float32"][b] - y64) / np.maximum(m, 1e-30))))
        _check_pcm16(got["pcm16"][b], y64, m)
        for enc in ("mulaw", "alaw"):
            assert np.array_equal(got[enc][b], tables[enc][got["pcm16"][b].astype(np.int64) + 32768]), (enc, b, n)
        if (up, down) == (1, 1):
            assert np.array_equal(got["float32"][b].view(np.int32), x.view(np.int32))
    _worst("audio_out_kernel err/m at %d Hz (bound %.3g)" % (rate, TAU), worst)
    f32 = got["float32"]
    order = list(range(len(lens)))[::-1]
    rev = abi_format(lib, dev, w, lens, up, down, "float32", items=order)
    for b, n in enumerate(lens):
        assert np.array_equal(rev[order.index(b)].view(np.int32), f32[b].view(np.int32)), b
        one = abi_format(lib, dev, np.ascontiguousarray(w[b:b + 1, :, :n + 5]), [n], up, down, "float32")[0]
        assert np.array_equal(one.view(np.int32), f32[b].view(np.int32)), (b, n)
    g = np.random.default_rng(rate + 1).uniform(0.25, 4.0, len(lens)).astype(np.float32)
    yg = abi_format(lib, dev, w, lens, up, down, "float32", gain=g)
    for b in range(len(lens)):
        assert np.array_equal(yg[b].view(np.int32), (f32[b] * g[b]).astype(np.float32).view(np.int32)), b


# ---- ev_limit ---------------------------------------------------------------------------------------------------------

def _limit_groups():
    """One representative rate per distinct (detector bank, hold) -> the representative rates sharing it."""
    groups = {}
    for rate in RATES:
        bank, hold = audio.limit_bank(SR, rate)
        groups.setdefault((bank.tobytes(), bank.shape, hold), []).append(rate)
    return {rates[0]: rates for rates in groups.values()}


LIMIT_GROUPS = _limit_groups()


def limit_items():
    """name -> float32 item at 16 kHz, loud enough to be limited: n around L and around the 1024-index tiles of n + L, and a
    long item whose level moves between 0 and +6 dBFS so every tile limits and releases."""
    L = audio.limit_lookahead(SR)
    rng = np.random.default_rng(77)
    lens = [1, L - 1, L, L + 1] + [e - L for e in (1023, 1024, 1025, 2047, 2048, 2049)]
    items = {"n%d" % n: (1.6 * np.tanh(rng.standard_normal(n))).astype(np.float32) for n in lens}
    n = 12 * 1024 + 333
    t = np.arange(n)
    env = 1.5 + 0.5 * np.sin(2 * np.pi * t / 2900.0)
    items["long"] = (env * np.tanh(rng.standard_normal(n))).astype(np.float32)
    return items


@pytest.mark.parametrize("rate", sorted(LIMIT_GROUPS))
def test_limiter_matches_the_oracle_at_every_bank(lib, dev, rate):
    items = limit_items()
    w, lens = padded_batch(list(items.values()))
    C = -1.0
    y = abi_limit(lib, dev, w, lens, rate, C)
    worst_rel = worst_db = 0.0
    for b, (name, x) in enumerate(items.items()):
        yo, Go, _ = LO.limit(x, SR, rate, C, 1.0)
        _compare(y[b, :lens[b]], x, 1.0, yo, Go, (name, rate))
        worst_rel = max(worst_rel, float(np.max(np.abs(y[b, :lens[b]].astype(np.float64) - yo) / np.maximum(np.abs(yo), 1e-30))))
        sel = np.abs(x) > 1e-3
        worst_db = max(worst_db, float(np.max(np.abs(20 * np.log10(y[b, :lens[b]][sel].astype(np.float64) / x[sel]) - Go[sel]))))
        assert np.all(np.isnan(y[b, lens[b]:])), name                         # nothing past the item is written
        if name == "long":
            tiles = [Go[s:s + 1024].min() for s in range(0, len(x), 1024)]
            assert max(tiles) < -0.5, (rate, np.round(tiles, 2))             # every tile limits
    _worst("lim_* at the bank of %s: sample rel (bound %g)" % (LIMIT_GROUPS[rate], REL), worst_rel)
    _worst("lim_* at the bank of %s: envelope dB (bound %g)" % (LIMIT_GROUPS[rate], ENV_DB), worst_db)


# ---- ev_loudness ------------------------------------------------------------------------------------------------------

LOUD_RATES = {8000: 1024, 16000: 2048, 48000: 6400}        # sr -> restart warm-up W


def abi_loudness_at(lib, dev, w, lens, sr, target=-23.0):
    """ev_loudness at ``sr`` straight through the ABI -> host (lufs, peak, gain) float32 arrays."""
    wt = torch.from_numpy(w).to(dev)
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    res = torch.empty((3, len(lens)), dtype=torch.float32, device=dev)
    kc = audio.k_weighting(sr)
    nb = lib.ev_loudness_workspace_bytes(len(lens), wt.stride(0), sr)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_loudness(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None, len(lens), sr, kc.ctypes.data, target,
                               res[0].data_ptr(), res[1].data_ptr(), res[2].data_ptr(), ws.data_ptr(), nb, _stream(dev)))
    r = res.cpu().numpy()
    return r[0], r[1], r[2]


def gate_margin_at(x, sr):
    """Smallest distance (LU) of a block's loudness to the absolute or relative gate (inf without blocks)."""
    _, l, rel = LU.gating(np.asarray(x, np.float64), sr)
    l = l[np.isfinite(l)]
    if not len(l):
        return np.inf
    m = np.abs(l + 70.0).min()
    return m if not np.isfinite(rel) else min(m, np.abs(l - rel).min())


def stepped(n, sr, seed):
    """Noise whose level alternates between -20 and -50 dBFS on 100 ms boundaries, so every block's loudness sits far from
    both gates: the blocks that hold some of a loud segment read above -27 LUFS, the others near -50, and the relative gate
    falls near -32 between them."""
    rng = np.random.default_rng(seed)
    S = sr // 10
    x = np.zeros(n)
    s, loud = 0, True
    while s < n:
        m = S * int(rng.integers(1, 13))
        x[s:s + m] = (0.1 if loud else 10 ** (-50 / 20)) * np.clip(rng.standard_normal(min(m, n - s)), -8, 8)
        s += m
        loud = not loud
    return x.astype(np.float32)


def loudness_items(sr):
    S = sr // 10
    items = {}
    for ns in (31, 32, 33, 128, 129, 257):
        items["sub%d" % ns] = stepped(ns * S, sr, ns)
        x = stepped(ns * S + 1, sr, ns + 1000)
        x[-1] = 0.95                                        # the peak is in the partial last sub-block
        items["sub%d+1" % ns] = x
    for nb in (255, 256, 257):
        items["blk%d" % nb] = stepped((nb + 3) * S, sr, nb + 2000)
    items["sine_1k_0dBFS"] = np.sin(2 * np.pi * 1000.0 * np.arange(5 * sr) / sr).astype(np.float32)
    return items


@pytest.mark.parametrize("sr", sorted(LOUD_RATES))
def test_loudness_matches_the_oracle_at_sub_block_and_block_edges(lib, dev, sr):
    assert audio.restart_warmup(audio.k_weighting(sr)) == LOUD_RATES[sr]
    items = loudness_items(sr)
    w, lens = padded_batch(list(items.values()))
    lufs, pk, g = abi_loudness_at(lib, dev, w, lens, sr)
    worst = 0.0
    for b, (name, x) in enumerate(items.items()):
        Lo = LU.integrated_loudness(x.astype(np.float64), sr)
        po = LU.peak(x)
        assert pk[b] == np.float32(po), (name, pk[b], po)
        if np.isfinite(Lo):
            assert gate_margin_at(x, sr) > 0.01, name
            assert abs(float(lufs[b]) - Lo) <= DL, (name, lufs[b], Lo)
            worst = max(worst, abs(float(lufs[b]) - Lo))
            go = LU.gain(Lo, po, -23.0)
            assert abs(g[b] / go - 1.0) <= 10.0 ** (DL / 20.0) - 1.0, (name, g[b], go)
        else:
            assert lufs[b] == -np.inf and g[b] == 1.0, (name, lufs[b])
    s = list(items).index("sine_1k_0dBFS")
    assert abs(float(lufs[s]) + 3.01) <= 0.1, lufs[s]
    _worst("loud_* at %d Hz: |L - L64| LU (bound %g)" % (sr, DL), worst)


# ---- ev_watermark_embed / ev_watermark_detect -------------------------------------------------------------------------

def embed_items():
    rng = np.random.default_rng(5)
    items = {}
    for i, n in enumerate((511, 512, 513, 3583, 3584, 3585, 7168, 7169)):
        x = speech_like(0.5, 200 + i)[:n] if i % 2 else (0.1 * rng.standard_normal(n)).astype(np.float32)
        items["n%d" % n] = x
    items["n40000"] = speech_like(2.5, 250)
    assert len(items["n40000"]) == 40000
    return items


def test_watermark_embed_matches_the_oracle_at_tile_edges_and_past_the_period(lib, dev):
    items = embed_items()
    w, lens = padded_batch(list(items.values()))
    y = abi_embed(lib, dev, w, lens)
    worst = 0.0
    for k, (name, x) in enumerate(items.items()):
        yo = W.embed(x.astype(np.float64), KEY)
        peak = max(float(np.max(np.abs(yo))), 1e-30)
        err = float(np.max(np.abs(y[k, :len(x)] - yo)))
        assert err <= EMBED_TOL * peak, (name, err, peak)
        assert np.all(np.isnan(y[k, len(x):])), name
        worst = max(worst, err / peak)
    assert W.n_frames(40000) == 80 and -(-40000 // W.H) == 79       # frames 0 .. 78 hold samples: the pattern wraps at 64
    _worst("wm_embed_kernel |y - y64| / peak (bound %g)" % EMBED_TOL, worst)


def _detect_against_the_oracle(z, off, ph, zt, mt, k, x):
    """-> (per-offset |best z - oracle's|, oracle's table); asserts the phases, z and the pick wherever Z_TOL decides them."""
    zo, tau, m0, table = W.detect(x.astype(np.float64), KEY)
    err = float(np.max(np.abs(zt[k] - table.max(axis=1))))
    top2 = np.sort(table, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * Z_TOL
    assert clear.sum() >= 0.9 * len(clear), (k, int(clear.sum()))
    flat = np.sort(table.ravel())
    print("detect item of %d samples: z %.4f (oracle %.4f) at (%d, %d) (oracle (%d, %d)); per-offset error %.3g"
          % (len(x), z[k], zo, off[k], ph[k], tau, m0, err))
    return err, clear, table, (zo, tau, m0, flat[-1] - flat[-2] > 2 * Z_TOL)


def test_watermark_detect_matches_the_full_search(lib, dev):
    """Marked noise of 40,000 samples (80 frames per offset: the fold wraps), 513 samples and 300 (shorter than a hop), held to
    Z_TOL; and a marked speech-like item of 40,000 samples, reported (see the module docstring)."""
    rng = np.random.default_rng(6)
    srcs = [(0.1 * rng.standard_normal(40000)).astype(np.float32), (0.1 * rng.standard_normal(513)).astype(np.float32),
            speech_like(2.5, 260)]
    w, lens = padded_batch(srcs, poison=False)
    marked = abi_embed(lib, dev, w, lens)
    xs = [marked[0, :40000], marked[1, :513], (0.1 * rng.standard_normal(300)).astype(np.float32), marked[2, :40000]]
    wc, lc = padded_batch(xs, poison=False)
    z, off, ph, zt, mt = abi_detect(lib, dev, wc[:, 0], lc)
    worst = 0.0
    for k, x in enumerate(xs[:3]):
        err, clear, table, (zo, tau, m0, decided) = _detect_against_the_oracle(z, off, ph, zt, mt, k, x)
        assert err <= Z_TOL, (k, err)
        assert np.array_equal(mt[k][clear], table.argmax(axis=1)[clear]), k
        assert abs(float(z[k]) - zo) <= Z_TOL, (k, z[k], zo)
        if decided:
            assert (off[k], ph[k]) == (tau, m0), (k, off[k], ph[k], tau, m0)
        worst = max(worst, err)
    _worst("wm_detect_kernel per-offset |z - z64| on noise (bound %g)" % Z_TOL, worst)
    err = _detect_against_the_oracle(z, off, ph, zt, mt, 3, xs[3])[0]
    _worst("wm_detect_kernel per-offset |z - z64| on 2.5 s of speech-like signal (reported)", err)


# ---- ev_flac_encode ---------------------------------------------------------------------------------------------------

def _check_flac(img, pcm, rate, what):
    want = F.encode(pcm, rate)
    assert img == want, (what, len(img), len(want), next((i for i, (a, b) in enumerate(zip(img, want)) if a != b), None))
    r, y, _ = F.decode(img)
    assert r == rate and np.array_equal(y, pcm), what


def flac_items():
    rng = np.random.default_rng(12)
    items = {}
    for n in (1, 256, 257, 4095, 4096, 4097, 8193):
        items["noise_%d" % n] = np.clip(np.round(rng.normal(0, 1500, n) + 4000 * np.sin(np.arange(n) * 0.03)), -32768,
                                        32767).astype(np.int16)
    items["silence"] = np.zeros(5000, np.int16)
    items["extremes"] = rng.choice(np.array([-32768, 32767], np.int16), 4100)
    return items


@pytest.mark.parametrize("rate", RATES)
def test_flac_matches_the_oracle_at_every_rate_code(model, lib, dev, rate):
    items = flac_items()
    for (name, x), img in zip(items.items(), abi_flac(lib, dev, list(items.values()), rate)):
        _check_flac(img, x, rate, (name, rate))
    lens = [1, 3001, 20000]
    w = _noise_batch(lens, rate + 7)
    out = out_dict(w, lens, dev)
    imgs = fd.fetch_audio(model, out, rate, "flac", hop=1)
    pcms = fd.fetch_audio(model, out, rate, "pcm16", hop=1)
    for b, (img, pcm) in enumerate(zip(imgs, pcms)):
        assert len(pcm) == audio.resampled_length(lens[b], *audio.plan(rate, "pcm16", SR)[1:])
        _check_flac(img.tobytes(), pcm, rate, ("fetch_audio", b, rate))
    code = audio.flac_rate_code(rate)[0]
    assert F.rate_code(rate)[0] == code
    print("flac at %d Hz (rate code %d): every image equals the oracle's" % (rate, code))


def long_speech(n, sr=SR, seed=2049):
    """int16 speech-like item of n samples: a gliding sawtooth source through three formant resonators, under a syllabic
    envelope, with pauses of digital silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f0 = 150.0 + 60.0 * np.sin(2 * np.pi * 0.3 * t) + 20.0 * np.sin(2 * np.pi * 2.1 * t)
    ph = np.cumsum(f0) / sr
    y = 2.0 * (ph - np.floor(ph)) - 1.0 + 0.05 * rng.standard_normal(n)
    for f, bw in ((700.0, 130.0), (1220.0, 70.0), (2600.0, 160.0)):
        r = np.exp(-np.pi * bw / sr)
        y = lfilter([1.0 - r], [1.0, -2.0 * r * np.cos(2 * np.pi * f / sr), r * r], y)
    y *= (0.1 + 0.9 * np.sqrt(np.maximum(0.0, np.sin(2 * np.pi * 3.7 * t)))) * (np.sin(2 * np.pi * t / 2.9) > -0.8)
    return np.round(y / np.abs(y).max() * 16000.0).astype(np.int16)


def test_flac_three_byte_frame_numbers_and_a_short_last_block(lib, dev):
    n = 2049 * 4096 + 257
    x = long_speech(n)
    assert len(F.utf8_number(2048)) == 3 and len(F.utf8_number(2047)) == 2
    img = abi_flac(lib, dev, [np.zeros(3, np.int16), x], 11025)[1]
    _check_flac(img, x, 11025, "long")
    frames = F.decode(img)[2]
    assert len(frames) == 2050
    print("%d samples at 11025 Hz: %d bytes, %.3f of PCM16" % (n, len(img), len(img) / (2 * n)))
