"""WORLD spectral envelopes and SPTK mel-cepstra on the GPU (``ev_world_envelope``, ``ev_sp2mc``, ``feats.spectral_envelope``,
``feats.sp2mc``, ``evaluate.compare(cepstrum="world")``, ``ev_eval_align``): the envelope against the fp64 oracle at 8, 16,
22.05, 24, 44.1 and 48 kHz with F0 of 0, on both sides of the floor, at 800 Hz and out of range, windows clamped at both item
ends, items of the shortest length and frames past each item's count; mel-cepstra from the envelope kernel and from ev_sp2mc
against the oracle's sp2mc; the same bits in any batch, order and NaN-poisoned padding and with EV_PDL=0; status bits;
a noise-free band-limited signal, whose quiet bands must stay positive and finite; ``compare(cepstrum="world")`` end to end
(itself, half the gain, noise-free signals, GPU mel-cepstra through the oracle's DTW, 48 kHz input against its 16 kHz
resampling, no host sync, launch counts) and argument errors on CUDA inputs.

The envelope bound (max |log sp_gpu - log sp_oracle|) and the mel-cepstrum bound were measured on an H100 80GB HBM3 and carry
a margin; the GPU's FFT and block sums round differently from the oracle's numpy FFT and sequential sums."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from conftest import ROOT
from emotivoice_b200 import _abi, evaluate, feats, recordings
from oracle import eval_oracle as O
from oracle import world_oracle as W
from test_evaluate_gpu import _host, _rows, speech

pytestmark = pytest.mark.gpu
RATES = [8000, 16000, 22050, 24000, 44100, 48000]
LOG_BOUND = 1e-11         # nepers, max over every bin of every frame; measured 2.9e-13 (16 kHz) to 8.2e-13 (48 kHz)
MC_BOUND = 1e-12          # absolute, on c0..c24; measured 7.1e-15 to 8.8e-15
QUIET_LOG_BOUND = 2e-7    # the same, on a noise-free band-limited signal; measured 2.9e-9 (16 kHz), 2.4e-8 (48 kHz)
QUIET_MC_BOUND = 1e-9     # measured 3.0e-11 (16 kHz), 9.5e-11 (48 kHz)


def voiced(n, fs, seed):
    """A seeded harmonic signal with a gliding F0 under a low noise floor, n samples at fs."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    f0 = 140.0 + 60.0 * np.sin(2 * np.pi * 2.0 * t + rng.uniform(0, 6.28))
    ph = 2 * np.pi * np.cumsum(f0) / fs
    x = sum(np.sin(h * ph) / h * (h * 200.0 < fs / 2) for h in range(1, 40))
    return (0.3 * x / np.abs(x).max() + 1e-3 * rng.standard_normal(n)).astype(np.float64)


def f0_track(F, fs, seed):
    """Per-frame F0 cycling through 0, just below and just above the floor, 71 Hz, speech values, 800 Hz, negative, above
    fs / 4 and NaN."""
    n_fft = W.fft_size(fs)
    fl = W.f0_floor(fs, n_fft)
    vals = [0.0, fl * 0.999, fl * 1.001, 71.0, 123.4, 220.0, 800.0, -5.0, fs / 4.0 + 1.0, math.nan, fs / 4.0, 310.0]
    rng = np.random.default_rng(seed)
    return np.array([vals[(i + int(rng.integers(len(vals)))) % len(vals)] for i in range(F)])


def run_envelope(lib, dev, items, fs, hop, f0s, table=None, with_sp=True, poison=True, status=False):
    """ev_world_envelope on items (host float64 arrays) with their F0 tracks, rows padded with NaN (or 0) past each item and
    F0 past each item's frames -> (sp, mc, status) on the host."""
    B = len(items)
    L = max(len(x) for x in items) + 37
    fp = feats.pitch_frame_period(fs, hop)
    F = feats.pitch_frames(L, fs, hop)
    fill = np.nan if poison else 0.0
    x = np.full((B, L), fill)
    f0 = np.full((B, F), fill)
    for b, it in enumerate(items):
        x[b, :len(it)] = it
        Fb = W.frame_count(len(it), fs, fp)
        f0[b, :Fb] = f0s[b][:Fb]
    xt, ft = torch.from_numpy(x).to(dev), torch.from_numpy(f0).to(dev)
    ns = torch.tensor([len(it) for it in items], dtype=torch.int64, device=dev)
    bins = W.fft_size(fs) // 2 + 1
    sp = torch.full((B, F, bins), 7.0, dtype=torch.float64, device=dev) if with_sp else None
    mc = None if table is None else torch.full((B, F, table.shape[0]), 7.0, dtype=torch.float64, device=dev)
    st = torch.zeros(1, dtype=torch.int32, device=dev) if status else None
    _abi.check(lib.ev_world_envelope(xt.data_ptr(), L, ns.data_ptr(), B, fs, fp, F, ft.data_ptr(), None if sp is None else sp.data_ptr(),
                                     None if table is None else table.data_ptr(), 0 if table is None else table.shape[0],
                                     None if mc is None else mc.data_ptr(), None if st is None else st.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    return (None if sp is None else sp.cpu().numpy(), None if mc is None else mc.cpu().numpy(), None if st is None else int(st.item()))


def rate_items(fs):
    """Three items at fs: the shortest length pitch_track takes, a short one and a longer one; hop of 5 ms."""
    hop = fs // 200
    lens = [feats.pitch_min_samples(fs), int(0.13 * fs) + 3, int(0.31 * fs)]
    items = [voiced(n, fs, 10 * i + fs % 97) for i, n in enumerate(lens)]
    fp = feats.pitch_frame_period(fs, hop)
    f0s = [f0_track(W.frame_count(n, fs, fp), fs, i) for i, n in enumerate(lens)]
    return hop, items, f0s


@pytest.mark.parametrize("fs", RATES)
def test_envelope_matches_the_oracle(lib, dev, fs):
    hop, items, f0s = rate_items(fs)
    fp = feats.pitch_frame_period(fs, hop)
    sp, _, st = run_envelope(lib, dev, items, fs, hop, f0s, status=True)
    assert st == 0
    worst = 0.0
    for b, it in enumerate(items):
        Fb = W.frame_count(len(it), fs, fp)
        want = W.cheaptrick(it, fs, f0s[b], fp, log=True)
        assert (sp[b, Fb:] == 0).all(), b                     # frames past the item's count
        got = np.log(sp[b, :Fb])
        assert np.isfinite(got).all(), b
        worst = max(worst, float(np.abs(got - want[:Fb]).max()))
    print("fs %d: max |log sp - oracle| = %.3e over %d frames" % (fs, worst, sum(W.frame_count(len(i), fs, fp) for i in items)))
    assert worst <= LOG_BOUND


@pytest.mark.parametrize("fs", [8000, 16000, 48000])
def test_mel_cepstra_of_the_envelope_kernel_and_of_ev_sp2mc(lib, dev, fs):
    hop, items, f0s = rate_items(fs)
    fp = feats.pitch_frame_period(fs, hop)
    n_fft = W.fft_size(fs)
    table = feats.mcep_table(n_fft, 24, 0.42, dev)
    sp, mc, _ = run_envelope(lib, dev, items, fs, hop, f0s, table=table)
    sp_only, mc_only, _ = run_envelope(lib, dev, items, fs, hop, f0s, table=table, with_sp=False)
    assert mc_only.tobytes() == mc.tobytes()
    worst_fused = worst_given = 0.0
    for b, it in enumerate(items):
        Fb = W.frame_count(len(it), fs, fp)
        assert (mc[b, Fb:] == 0).all()
        want_sp = W.cheaptrick(it, fs, f0s[b], fp)[:Fb]
        want = np.stack([W.sp2mc(s, 24, 0.42) for s in want_sp])
        worst_fused = max(worst_fused, float(np.abs(mc[b, :Fb] - want).max()))
        given = feats.sp2mc(torch.from_numpy(want_sp).to(dev), 24, 0.42).cpu().numpy()
        worst_given = max(worst_given, float(np.abs(given - want).max()))
    print("fs %d: mel-cepstra max abs error %.3e (envelope kernel), %.3e (ev_sp2mc on the oracle's envelopes)"
          % (fs, worst_fused, worst_given))
    assert worst_fused <= MC_BOUND
    assert worst_given <= 1e-12


def band_limited(n, fs, f0=93.2, top=4000.0, seed=0):
    """A noise-free harmonic signal: F0 f0, harmonics up to top Hz with seeded phases, rounded to float32 as compare's
    inputs are.  Above top its spectrum is only the window's leakage, far below the power of the harmonics."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    x = sum(np.sin(2 * np.pi * h * f0 * t + rng.uniform(0, 6.28)) / h for h in range(1, int(top / f0) + 1))
    return (0.5 * x / np.abs(x).max()).astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_noise_free_band_limited_signal(lib, dev, fs):
    """Bands with no signal are where a difference of two running sums of the whole spectrum would cancel to nothing or to
    a negative value; the smoothing's local sums keep every bin positive and the envelope finite."""
    hop = fs // 200
    items = [band_limited(int(0.4 * fs), fs), band_limited(int(0.25 * fs) + 11, fs, f0=131.0, top=3000.0, seed=1)]
    fp = feats.pitch_frame_period(fs, hop)
    f0s = []
    for b, it in enumerate(items):
        f = np.full(W.frame_count(len(it), fs, fp), 93.2 if b == 0 else 131.0)
        f[::7] = 0.0                                          # some frames at the 500 Hz default
        f0s.append(f)
    table = feats.mcep_table(W.fft_size(fs), 24, 0.42, dev)
    sp, mc, st = run_envelope(lib, dev, items, fs, hop, f0s, table=table, status=True)
    assert st == 0
    worst = worst_mc = 0.0
    for b, it in enumerate(items):
        Fb = W.frame_count(len(it), fs, fp)
        assert np.isfinite(sp[b]).all() and (sp[b, :Fb] > 0).all() and np.isfinite(mc[b]).all(), b
        want = W.cheaptrick(it, fs, f0s[b], fp, log=True)
        worst = max(worst, float(np.abs(np.log(sp[b, :Fb]) - want).max()))
        want_mc = np.stack([W.sp2mc(np.exp(v), 24, 0.42) for v in want])
        worst_mc = max(worst_mc, float(np.abs(mc[b, :Fb] - want_mc).max()))
        print("fs %d item %d: envelope from %.3e to %.3e" % (fs, b, sp[b, :Fb].min(), sp[b, :Fb].max()))
    print("fs %d noise-free: max |log sp - oracle| = %.3e, mel-cepstra %.3e" % (fs, worst, worst_mc))
    assert worst <= QUIET_LOG_BOUND and worst_mc <= QUIET_MC_BOUND


def test_world_compare_of_noise_free_signals_is_finite(dev):
    x = band_limited(48000, 16000)
    y = band_limited(52000, 16000, f0=98.0, seed=3)
    xs = [x.astype(np.float32), y.astype(np.float32)]
    c = _host(evaluate.compare(_rows(xs, dev), _rows(xs[::-1], dev), syn_lengths=[len(v) for v in xs],
                               ref_lengths=[len(v) for v in xs[::-1]], cepstrum="world"))
    print("noise-free world mcd %s" % c["mcd"])
    assert np.isfinite(c["mcd"]).all() and (c["mcd"] > 0).all()
    self_ = _host(evaluate.compare(_rows(xs, dev), _rows(xs, dev), cepstrum="world", syn_lengths=[len(v) for v in xs],
                                   ref_lengths=[len(v) for v in xs]))
    assert (self_["mcd"] == 0).all()


def _mixed(fs=16000):
    hop = 80
    lens = [feats.pitch_min_samples(fs), 4000, 9000, 1500, 6001]
    items = [voiced(n, fs, 40 + i) for i, n in enumerate(lens)]
    items[3] = np.zeros(lens[3])                              # digital silence
    f0s = [f0_track(W.frame_count(n, fs, feats.pitch_frame_period(fs, hop)), fs, 50 + i) for i, n in enumerate(lens)]
    return hop, items, f0s


def test_batch_order_and_poison_do_not_change_any_bit(lib, dev):
    hop, items, f0s = _mixed()
    table = feats.mcep_table(1024, 24, 0.42, dev)
    sp, mc, _ = run_envelope(lib, dev, items, 16000, hop, f0s, table=table)
    assert np.isfinite(sp).all() and np.isfinite(mc).all()
    zeros = run_envelope(lib, dev, items, 16000, hop, f0s, table=table, poison=False)
    rev = run_envelope(lib, dev, items[::-1], 16000, hop, f0s[::-1], table=table)
    for b in range(len(items)):
        alone = run_envelope(lib, dev, [items[b]], 16000, hop, [f0s[b]], table=table)
        F = alone[0].shape[1]
        for other_sp, other_mc in ((sp[b], mc[b]), (zeros[0][b], zeros[1][b]), (rev[0][len(items) - 1 - b], rev[1][len(items) - 1 - b])):
            assert other_sp[:F].tobytes() == alone[0][0].tobytes(), b
            assert other_mc[:F].tobytes() == alone[1][0].tobytes(), b
            assert (other_sp[F:] == 0).all() and (other_mc[F:] == 0).all(), b


def test_status_bits(lib, dev):
    fs, hop = 16000, 160
    good = voiced(4000, fs, 1)
    bad = good.copy()
    bad[3999] = np.inf
    f0s = [np.full(30, 150.0)] * 2
    assert run_envelope(lib, dev, [good, bad], fs, hop, f0s, status=True)[2] == 1
    short = good[:feats.pitch_min_samples(fs) - 1]
    sp, _, st = run_envelope(lib, dev, [good, short], fs, hop, f0s, status=True)
    assert st == 2 and (sp[1] == 0).all() and (sp[0, 0] > 0).all()


def pdl_dump(path):
    """Envelopes, mel-cepstra and compare(cepstrum="world") of fixed inputs (run under EV_PDL=0 below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    dev = torch.device("cuda:0")
    lib = _abi.load()
    hop, items, f0s = _mixed()
    sp, mc, _ = run_envelope(lib, dev, items, 16000, hop, f0s, table=feats.mcep_table(1024, 24, 0.42, dev))
    out = {"sp": sp, "mc": mc}
    syn, ref, ls, lr = _pair(dev)
    c = evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True, cepstrum="world")
    out.update({k: getattr(c, k).cpu().numpy() for k in c._fields})
    np.savez(path, **out)


def test_same_bits_with_pdl_off(tmp_path):
    here, off = str(tmp_path / "on.npz"), str(tmp_path / "off.npz")
    pdl_dump(here)
    py = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(py), EV_PDL="0")
    subprocess.run([sys.executable, "-c", "import test_world_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=900)
    x, y = np.load(here), np.load(off)
    assert sorted(x.files) == sorted(y.files)
    for k in x.files:
        assert x[k].tobytes() == y[k].tobytes(), k


def test_spectral_envelope_and_sp2mc_api(dev):
    fs, hop = 22050, 256
    w = [voiced(7000, fs, 3), voiced(5000, fs, 4)]
    x = torch.zeros((2, 7100), dtype=torch.float32, device=dev)
    for b, it in enumerate(w):
        x[b, :len(it)] = torch.from_numpy(it.astype(np.float32))
    lens = [7000, 5000]
    F = feats.pitch_frames(7100, fs, hop)
    sp = feats.spectral_envelope(x, fs, hop, lengths=lens)
    assert sp.shape == (2, F, 513) and sp.dtype == torch.float64
    f0 = feats.pitch_track(x, fs, hop, continuous=False, lengths=lens)
    assert torch.equal(feats.spectral_envelope(x, fs, hop, f0=f0, lengths=lens), sp)
    mc = feats.sp2mc(sp[:, :10], 30, 0.45)
    assert mc.shape == (2, 10, 31)
    flat = feats.sp2mc(sp[:, :10].reshape(20, 513), 30, 0.45)
    assert torch.equal(flat.reshape(2, 10, 31), mc)
    for bad_f0 in (f0[:, :-1], f0.float(), f0.cpu()):
        with pytest.raises(ValueError):
            feats.spectral_envelope(x, fs, hop, f0=bad_f0, lengths=lens)
    with pytest.raises(ValueError):
        feats.spectral_envelope(x, fs, hop, lengths=[feats.pitch_min_samples(fs) - 1, 5000])
    with pytest.raises(ValueError):
        feats.spectral_envelope(x, 7999, hop)
    for bad in (sp[..., :512], sp.float(), torch.ones((3, 4097), dtype=torch.float64, device=dev)):
        with pytest.raises(ValueError):
            feats.sp2mc(bad, 24, 0.42)


# ---- compare(cepstrum="world") -----------------------------------------------------------------------------------------------
def _pair(dev):
    syn = [speech(3.0, 1), speech(5.5, 2)]
    ref = [speech(3.2, 4, semitones=1.0), speech(5.5, 2) * np.float32(0.5)]
    return _rows(syn, dev), _rows(ref, dev), [len(x) for x in syn], [len(x) for x in ref]


def test_world_against_itself_and_half_the_gain(dev):
    x = speech(6.0, 3)
    half = x * np.float32(0.5)
    n = [len(x)] * 2
    N = len(x) // 256 + 1
    c = _host(evaluate.compare(_rows([x, x], dev), _rows([x, half], dev), syn_lengths=n, ref_lengths=n, return_path=True,
                               cepstrum="world"))
    print("world: itself mcd %g; x 0.5: mcd %.3g dB, vuv %.4f" % (c["mcd"][0], c["mcd"][1], c["vuv_error"][1]))
    assert c["mcd"][0] == 0.0 and c["vuv_error"][0] == 0.0 and c["f0_rmse"][0] == 0.0
    assert np.array_equal(c["path"][0, :N], np.stack([np.arange(N)] * 2, axis=1))
    assert c["mcd"][1] < 0.01
    mel = _host(evaluate.compare(_rows([x, x], dev), _rows([x, half], dev), syn_lengths=n, ref_lengths=n, return_path=True))
    dflt = _host(evaluate.compare(_rows([x, x], dev), _rows([x, half], dev), syn_lengths=n, ref_lengths=n, return_path=True,
                                  cepstrum="mel"))
    for k in mel:
        assert mel[k].tobytes() == dflt[k].tobytes(), k


def test_gpu_mel_cepstra_fed_to_the_oracle_dtw_give_the_same_results(dev):
    syn, ref, ls, lr = _pair(dev)
    c = _host(evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True, cepstrum="world", alpha=0.42))
    table = feats.mcep_table(1024, 24, 0.42, dev, first=1)
    cs, fs = (t.cpu().numpy() for t in evaluate._world_features(syn, ls, table))
    cr, fr = (t.cpu().numpy() for t in evaluate._world_features(ref, lr, table))
    for b in range(len(ls)):
        N, M = ls[b] // 256 + 1, lr[b] // 256 + 1
        d = O.distances(cs[b, :N], cr[b, :M])
        _, code = O.dtw(d)
        path = O.backtrack(code)
        want = O.statistics(d, path, fs[b, :N], fr[b, :M])
        P = int(c["path_length"][b])
        assert P == want["path_length"] and np.array_equal(c["path"][b, :P], path), b
        assert int(c["voiced_pairs"][b]) == want["voiced_pairs"]
        for k in ("mcd", "f0_rmse", "vuv_error"):
            assert abs(float(c[k][b]) - want[k]) <= 1e-12 * abs(want[k]), (b, k)
        print("pair %d: world mcd %.4f dB over P %d" % (b, c["mcd"][b], P))
    other = _host(evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, cepstrum="world", alpha=0.3))
    assert not np.array_equal(other["mcd"], c["mcd"])


def test_world_48k_input_gives_the_bits_of_its_16k_resampling(dev):
    xs = [resample_poly(speech(2.5, 7), 3, 1).astype(np.float32), resample_poly(speech(4.0, 8), 3, 1).astype(np.float32)]
    ys = [resample_poly(speech(2.7, 9), 3, 1).astype(np.float32), resample_poly(speech(4.0, 8, semitones=1.0), 3, 1).astype(np.float32)]
    s48, r48 = _rows(xs, dev), _rows(ys, dev)
    ls, lr = [len(x) for x in xs], [len(y) for y in ys]
    a = _host(evaluate.compare(s48, r48, sample_rate=48000, syn_lengths=ls, ref_lengths=lr, return_path=True, cepstrum="world"))
    s16, ls16 = recordings.resample(s48.contiguous(), ls, 48000, 16000)
    r16, lr16 = recordings.resample(r48.contiguous(), lr, 48000, 16000)
    b = _host(evaluate.compare(s16, r16, syn_lengths=ls16, ref_lengths=lr16, return_path=True, cepstrum="world"))
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_world_compare_does_not_wait_for_the_device_and_counts_its_launches(dev):
    syn, ref, ls, lr = _pair(dev)
    call = lambda: evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True, cepstrum="world")   # noqa: E731
    call()                                                    # the first call on a device builds its tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        call()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    feats.pitch_track(syn, 16000, 256, continuous=False, lengths=ls)
    n_pitch = _abi.launch_count() - n0
    n0 = _abi.launch_count()
    call()
    assert _abi.launch_count() == n0 + 2 * (n_pitch + 1) + 2
    n0 = _abi.launch_count()
    for kw in (dict(cepstrum="sptk"), dict(cepstrum=None), dict(alpha=0.42), dict(cepstrum="world", alpha=1.0),
               dict(cepstrum="world", alpha=-1.0), dict(cepstrum="world", alpha="0.42"), dict(cepstrum="world", alpha=True),
               dict(cepstrum="world", alpha=float("nan"))):
        with pytest.raises(ValueError):
            evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, **kw)
    assert _abi.launch_count() == n0


def test_abi_argument_errors(lib, dev):
    x = torch.zeros((1, 4000), dtype=torch.float64, device=dev)
    f0 = torch.zeros((1, 26), dtype=torch.float64, device=dev)
    sp = torch.empty((1, 26, 513), dtype=torch.float64, device=dev)
    table = feats.mcep_table(1024, 24, 0.42, dev)
    mc = torch.empty((1, 26, 25), dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    n0 = _abi.launch_count()

    def env(xp=x.data_ptr(), L=4000, B=1, fs=16000, fp=10.0, F=26, fp0=f0.data_ptr(), spp=sp.data_ptr(), tp=table.data_ptr(), n_out=25,
            mcp=mc.data_ptr()):
        return lib.ev_world_envelope(xp, L, None, B, fs, fp, F, fp0, spp, tp, n_out, mcp, None, st)

    for kw in (dict(xp=None), dict(fp0=None), dict(spp=None, mcp=None), dict(B=0), dict(fs=7999), dict(fs=48001), dict(fp=0.2),
               dict(F=25), dict(tp=None), dict(n_out=0), dict(n_out=257), dict(L=640, F=5)):
        assert env(**kw) == -1, kw
    assert _abi.launch_count() == n0
    assert env() == 0 and env(mcp=None) == 0 and env(spp=None) == 0
    assert _abi.launch_count() == n0 + 3
    n0 = _abi.launch_count()
    for bins, n_out, frames in ((512, 25, 26), (2050, 25, 26), (513, 0, 26), (513, 257, 26), (513, 25, -1)):
        assert lib.ev_sp2mc(sp.data_ptr(), frames, bins, table.data_ptr(), n_out, mc.data_ptr(), st) == -1, (bins, n_out, frames)
    assert lib.ev_sp2mc(sp.data_ptr(), 0, 513, table.data_ptr(), 25, mc.data_ptr(), st) == 0
    assert _abi.launch_count() == n0
    cep = torch.zeros((1, 32, 24), dtype=torch.float64, device=dev)
    f0a = torch.zeros((1, 32), dtype=torch.float64, device=dev)
    cnt = torch.tensor([20, 30], dtype=torch.int32, device=dev)
    stats = torch.empty((3, 1), dtype=torch.float64, device=dev)
    co = torch.empty((2, 1), dtype=torch.int32, device=dev)
    nb = lib.ev_eval_workspace_bytes(1, 20, 30)
    ws = torch.empty((nb,), dtype=torch.uint8, device=dev)

    def align(cp=cep.data_ptr(), k=1, frames=32, max_n=20, wsb=nb):
        return lib.ev_eval_align(cp, f0a.data_ptr(), frames, cnt.data_ptr(), max_n, cep.data_ptr(), f0a.data_ptr(), 32, cnt.data_ptr() + 4,
                                 30, k, stats.data_ptr(), co.data_ptr(), None, 0, ws.data_ptr(), wsb, st)

    for kw in (dict(cp=None), dict(k=0), dict(frames=19), dict(max_n=4097), dict(wsb=nb - 1)):
        assert align(**kw) == -1, kw
    assert _abi.launch_count() == n0
    assert align() == 0 and _abi.launch_count() == n0 + 2
