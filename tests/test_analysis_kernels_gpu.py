"""The recording-analysis kernels against their fp64 oracles at every class of what the analysis API accepts
(tests/analysis_plans.py): ``stft_feats_kernel`` through TacotronSTFT, mel_spectrogram_torch and Energy at every representative
rate, basis and hop, frame counts around the 32-frame tile, the shortest items and the reference-default objects; ``ev_pitch``
at every representative rate around both FIR tile edges, at the hop edges, at StoneMask's fs / 12 gate and FFT-size step, where
pyworld's frame count is not n // hop + 1, and at Pitch()'s defaults; ``ev_world_envelope`` at the hop edges and the
mel-cepstra of it and of ``ev_sp2mc`` at every representative output-row count, bin count and alpha; ``ev_eval_align`` called
directly with row strides past the longest item.  Batches with NaN past each item are bitwise their single calls.

The bounds are the existing files' (test_feats_gpu's log-mel and energy bounds, test_pitch_gpu's 1e-8 with identical voicing,
test_world_gpu's LOG_BOUND and MC_BOUND, test_evaluate_gpu's bitwise paths and 1e-12 statistics), except where MC_BOUND was
never measured: at order 255 and near |alpha| = 1 the mel-cepstrum bound is

    (n_fft + bins + order + 1) 2^-52 max_k sum_n |T[k, n] log sp[n]|       (per frame, T the sp2mc table)

a first-order count of the roundings on each side: the kernel's bins-term dot product of each row (at most bins 2^-52 of that
row's sum of |products|), and the freqt recursion, which the table's columns and the oracle's coefficients both run over n_fft
coefficients with up to order + 1 terms per step, each rounded to the magnitude of the frame's largest row sum.  Each test prints
its worst error per class against its bound and its time.

Measured on an H100 80GB HBM3 (700 W power limit), the whole file in 65 s: log-mel and energy at most 0.115 of their bounds
(the 8 kHz basis with 17 empty bands, and 128 bands at 48 kHz); every pitch track within 1e-8 with identical voicing; the
envelope at the hop edges 3.5e-13 (8 kHz, hop 16) to 1.4e-12 nepers (48 kHz, hop 16), above the 8.2e-13 test_world_gpu
records at a 5 ms hop and under LOG_BOUND; mel-cepstra at alpha 0.42 up to 33 rows 7.4e-15 (envelope kernel) and 8.9e-16
(ev_sp2mc), at 256 rows 7.4e-15, at most 0.0013 of the derived bound; at alpha -0.99 and 0.99 1.6e-14, at most 0.13 of the
derived bound (3 bins, one row); ev_eval_align's statistics equal to the oracle's at every shape.
"""
import math
import time

import numpy as np
import pytest
import torch

import analysis_plans as P
from emotivoice_b200 import _abi, align, feats
from oracle import eval_oracle as O
from oracle import feats_oracle as FO
from oracle import pitch_oracle as PO
from oracle import world_oracle as W
from test_evaluate_gpu import SHAPES, _rel
from test_feats_gpu import _energy_bound, _logmel_bound
from test_pitch_gpu import REL, _voice, check_track, gpu
from test_world_gpu import LOG_BOUND, MC_BOUND, f0_track, run_envelope, voiced

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -52


@pytest.fixture(autouse=True)
def _section_time(request):
    t0 = time.time()
    yield
    print("[%s: %.1f s]" % (request.node.name, time.time() - t0))


# ---- stft_feats_kernel -------------------------------------------------------------------------------------------------------
def _signal(n, sr, seed):
    """Two tones at 4 % and 18 % of the rate and a little noise, in [-1, 1]."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.4 * np.sin(2 * np.pi * 0.04 * sr * t) + 0.2 * np.sin(2 * np.pi * 0.18 * sr * t + 1.0) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def _basis(sr, n_mels, fmin, fmax):
    return feats.mel_filterbank(sr=sr, n_fft=1024, n_mels=n_mels, fmin=fmin, fmax=fmax)


def stft_run(case, y, lengths=None):
    """-> log-mel (B, n_mels, F) or energy (B, F) of one call, as numpy."""
    variant, sr, n_mels, fmin, fmax, hop = case
    yt = torch.from_numpy(np.atleast_2d(np.asarray(y, np.float32))).to(DEV)
    if variant == "taco":
        stft = feats.TacotronSTFT(hop_length=hop, n_mel_channels=n_mels, sampling_rate=sr, mel_fmin=fmin, mel_fmax=fmax)
        return stft.to(DEV).mel_spectrogram(yt, lengths=lengths).cpu().numpy()
    if variant == "mt":
        return feats.mel_spectrogram_torch(yt, 1024, n_mels, sr, hop, 1024, fmin, fmax, lengths=lengths).cpu().numpy()
    return feats.Energy(sr=sr, n_fft=1024, hop_length=hop).get_energy(yt, lengths=lengths).cpu().numpy()


def stft_check(case, y, got):
    """got (one item's output) against fp64 -> worst err / bound; asserts every element is within the bound."""
    variant, sr, n_mels, fmin, fmax, hop = case
    if variant == "energy":
        r64 = FO.features64(y, 512, hop, feats.hann_window_scipy(), 0.0, np.zeros((1, 513)))
        err, bnd = np.abs(got - r64["energy"]), _energy_bound(r64)
    else:
        basis = _basis(sr, n_mels, fmin, fmax)
        r64 = FO.tacotron64(y, hop, basis) if variant == "taco" else FO.mel_spectrogram64(y, hop, basis)
        err, bnd = np.abs(got - r64["logmel"]), _logmel_bound(r64, basis)
    assert err.shape == bnd.shape, (case, err.shape, bnd.shape)
    bad = err > bnd
    assert not bad.any(), "%s n=%d: %d elements over the bound, worst err %.3e vs bound %.3e" % (
        case, len(y), int(bad.sum()), float(err[bad].max()), float(bnd[bad][np.argmax(err[bad])]))
    return float((err / bnd).max())


def stft_lengths(case):
    """n = pad + 1, the frame counts 31, 32, 33 and 65 where an item that long exists, otherwise the first tile edges
    (32k - 1, 32k, 32k + 1, 32(k + 1) + 1) past the shortest item."""
    variant, hop = case[0], case[5]
    pad = P.pad_of(variant, hop)
    shortest = pad + 1 if pad + 1 + 2 * pad >= 1024 else 1024 - 2 * pad
    fmin = feats.n_frames(shortest, pad, hop)
    k = max(1, -(-fmin // P.TILE))
    counts = [31, 32, 33, 65] if fmin <= 31 else [P.TILE * k - 1, P.TILE * k, P.TILE * k + 1, P.TILE * (k + 1) + 1]
    ns = [shortest] + [(f - 1) * hop + 1024 - 2 * pad for f in counts if f >= fmin]
    return ns, counts


@pytest.mark.parametrize("case", [c for c, _ in P.STFT_CASES], ids=lambda c: "%s-%d-%s-%s-%s-hop%d" % c)
def test_stft_against_fp64_at_every_representative(case):
    ns, counts = stft_lengths(case)
    worst = 0.0
    for i, n in enumerate(ns):
        y = _signal(n, case[1], 7000 + i)
        out = stft_run(case, y)
        assert out.shape[-1] == feats.n_frames(n, P.pad_of(case[0], case[5]), case[5])
        worst = max(worst, stft_check(case, y, out[0]))
    fmin = feats.n_frames(ns[0], P.pad_of(case[0], case[5]), case[5])
    assert [feats.n_frames(n, P.pad_of(case[0], case[5]), case[5]) for n in ns[1:]] == [f for f in counts if f >= fmin]
    print("stft %s: worst err / bound %.3f over lengths %s" % (case, worst, ns))


def test_stft_reference_default_objects():
    stft = feats.TacotronSTFT().to(DEV)
    assert (stft.sampling_rate, stft.hop_length, stft.n_mel_channels) == (22050, 256, 80)
    en = feats.Energy(sr=24000, n_fft=1024, hop_length=300)
    worst = 0.0
    for i, n in enumerate([22050, 22050 // 3 + 17]):
        y = _signal(n, 22050, 7100 + i)
        got = stft.mel_spectrogram(torch.from_numpy(y)[None].to(DEV)).cpu().numpy()
        assert got.shape == (1, 80, n // 256 + 1)
        worst = max(worst, stft_check(("taco", 22050, 80, 0.0, 8000.0, 256), y, got[0]))
        y = _signal(n + 1950, 24000, 7200 + i)
        e = en.get_energy(torch.from_numpy(y).to(DEV)).cpu().numpy()
        assert e.shape == (len(y) // 300 + 1,)
        worst = max(worst, stft_check(("energy", 24000, None, None, None, 300), y, e))
    print("reference defaults: worst err / bound %.3f" % worst)


@pytest.mark.parametrize("hop", [1, 1024])
@pytest.mark.parametrize("variant", ["taco", "mt", "energy"])
def test_stft_nan_padded_batch_is_bitwise_its_items(variant, hop):
    case = (variant, 48000, 128, 0.0, 8000.0, hop) if variant != "energy" else ("energy", 48000, None, None, None, hop)
    pad = P.pad_of(variant, hop)
    shortest = max(pad + 1, 1024 - 2 * pad)
    lens = [shortest, 1500, 1100, 700 + pad] if hop == 1 else [shortest, 20000, 5000, 3071]
    N = max(lens)
    y = np.full((len(lens), N), np.nan, np.float32)
    items = [_signal(n, 48000, 7300 + b) for b, n in enumerate(lens)]
    for b, it in enumerate(items):
        y[b, :len(it)] = it
    out = stft_run(case, y, lengths=lens)
    assert out.shape[-1] == feats.n_frames(N, pad, hop) and np.isfinite(out).all()
    for b, n in enumerate(lens):
        one = stft_run(case, items[b])[0]
        fb = feats.n_frames(n, pad, hop)
        assert one.shape[-1] == fb and np.array_equal(out[b][..., :fb], one), (b, n)
        assert (out[b][..., fb:] == 0.0).all(), b


# ---- ev_pitch ----------------------------------------------------------------------------------------------------------------
def _oracle(x, fs, hop):
    f0, t = PO.dio(x, fs, feats.pitch_frame_period(fs, hop))
    return f0, PO.stonemask(x, f0, t, fs)


def pitch_against_oracle(items, fs, hop, what, batch=True):
    """items run as one NaN-padded batch (or one call each) -> each item's DIO and StoneMask tracks checked against the
    oracle's; -> the number of voiced frames."""
    if batch:
        N = max(len(x) for x in items)
        rows = np.full((len(items), N), np.nan)
        for b, x in enumerate(items):
            rows[b, :len(x)] = x
        out, f0 = gpu(rows, fs, hop, lengths=[len(x) for x in items])
        assert out.shape == (len(items), feats.pitch_frames(N, fs, hop))
    voiced_frames = 0
    for b, x in enumerate(items):
        if not batch:
            o1, f1 = gpu(x, fs, hop)
        else:
            o1, f1 = out[b:b + 1], f0[b:b + 1]
        Fb = feats.pitch_frames(len(x), fs, hop)
        assert Fb == PO.frame_count(len(x), fs, feats.pitch_frame_period(fs, hop))
        assert not o1[0, Fb:].any() and not f1[0, Fb:].any()
        f0w, refw = _oracle(x, fs, hop)
        check_track(f1[0, :Fb], f0w, x, fs, hop, "dio %s n=%d" % (what, len(x)))
        check_track(o1[0, :Fb], refw, x, fs, hop, "stonemask %s n=%d" % (what, len(x)))
        voiced_frames += int((refw > 0).sum())
    return voiced_frames


def rate_lengths(fs):
    """pitch_min_samples, the 256-sample FIR tile edges of n + 1 (band filters) and of n + 1 + 2 l0 (low-cut), about 1 s."""
    m = feats.pitch_min_samples(fs)
    l0 = max(P.band_halves(fs))
    k = -(-(m + 1) // 256) + 1
    ns = [m] + [256 * k + d - 1 for d in (-1, 0, 1)]
    k2 = -(-(m + 1 + 2 * l0) // 256) + 1
    ns += [256 * k2 + d - 1 - 2 * l0 for d in (-1, 0, 1)]
    return ns + [fs + 123]


@pytest.mark.parametrize("fs", sorted(P.PITCH_RATE_CASES))
def test_pitch_at_every_representative_rate(fs):
    hop = P.PITCH_RATE_CASES[fs][0]
    ns = rate_lengths(fs)
    assert min(ns) >= feats.pitch_min_samples(fs)
    items = [_voice(n, fs, 100 + i, f0=140.0 + 10 * i) for i, n in enumerate(ns)]
    v = pitch_against_oracle(items, fs, hop, "fs %d" % fs)
    print("pitch fs %d hop %d: lengths %s, %d voiced frames within 1e-8" % (fs, hop, ns, v))
    assert v > 0


@pytest.mark.parametrize("fs,hop", P.PITCH_HOP_EDGES)
def test_pitch_at_the_hop_edges(fs, hop):
    ns = [feats.pitch_min_samples(fs), int(0.2 * fs)] if hop == 16 else [int(1.5 * fs) + 11, 3 * fs if fs == 8000 else 2 * fs]
    items = [_voice(n, fs, 200 + i) for i, n in enumerate(ns)]
    v = pitch_against_oracle(items, fs, hop, "fs %d hop %d" % (fs, hop))
    print("pitch fs %d hop %d (r = %d): %d voiced frames" % (fs, hop, P.fix_width(fs, hop), v))
    assert v > 0


def test_pitch_bands_with_fewer_than_four_events():
    fs, hop = 8000, 16
    x = _voice(feats.pitch_min_samples(fs), fs, 5)
    _, _, det = PO.dio(x, fs, feats.pitch_frame_period(fs, hop), details=True)
    least = det["counts"].min(axis=1)
    assert (least <= 3).any() and (least > 3).any(), least     # both sides of the cnt - 3 > 0 gate
    pitch_against_oracle([x], fs, hop, "few events", batch=False)


def test_pitch_stonemask_gate_at_8k():
    """A voice at 710-780 Hz: DIO finds it (ceiling 800 Hz), StoneMask leaves every frame above fs / 12 = 666.7 Hz at 0."""
    fs, hop = 8000, 80
    x = _voice(fs, fs, 7, f0=740.0)
    f0w, refw = _oracle(x, fs, hop)
    assert (f0w > fs / 12.0).sum() > 50 and not refw[f0w > fs / 12.0].any()
    pitch_against_oracle([x, _voice(fs // 2, fs, 8, f0=620.0)], fs, hop, "stonemask gate")


def _tone(n, fs, f0, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    return sum(0.3 / k * np.sin(2 * np.pi * k * f0 * t + k) for k in range(1, 6)) + 1e-4 * rng.standard_normal(n)


def test_pitch_either_side_of_a_stonemask_fft_size_step():
    """At 16 kHz StoneMask's FFT size 2^(2 + int(log2(1.5 fs / f0 + 1))) steps from 1024 to 512 at f0 = 94.1 Hz."""
    fs, hop = 16000, 256
    size = lambda f: 2 ** (2 + int(math.log(1.5 * fs / f + 1.0) / PO.LOG2))     # noqa: E731
    items = [_tone(fs, fs, 92.0, 1), _tone(fs, fs, 97.0, 2)]
    for x, want in zip(items, (1024, 512)):
        f0w, _ = _oracle(x, fs, hop)
        assert {size(f) for f in f0w[f0w > 0]} == {want}
    pitch_against_oracle(items, fs, hop, "fft-size step")


def test_pitch_where_pyworlds_frame_count_is_not_n_over_hop_plus_1():
    (fs, hop), ns = next(iter(P.FRAME_COUNT_LENGTHS.items()))
    items = [_voice(n, fs, 300 + i) for i, n in enumerate(ns)]
    for x in items:
        assert feats.pitch_frames(len(x), fs, hop) == len(x) // hop
    pitch_against_oracle(items, fs, hop, "frame count", batch=False)
    L = max(ns) + 1000
    rows = np.full((len(items), L), np.nan)
    for b, x in enumerate(items):
        rows[b, :len(x)] = x
    bo, bf = gpu(rows, fs, hop, lengths=ns)
    assert bo.shape[1] == feats.pitch_frames(L, fs, hop)
    for b, x in enumerate(items):
        so, sf = gpu(x, fs, hop)
        Fb = so.shape[1]
        assert Fb == PO.frame_count(len(x), fs, feats.pitch_frame_period(fs, hop))
        assert np.array_equal(bo[b, :Fb], so[0]) and np.array_equal(bf[b, :Fb], sf[0]) and not bo[b, Fb:].any()


def test_pitch_at_the_reference_defaults():
    Pt = feats.Pitch()
    fs, hop = Pt.sr, Pt.hop_length
    assert (fs, hop) == (24000, 300)
    x = _voice(int(1.5 * fs), fs, 400, f0=160.0)
    f0w, refw = _oracle(x, fs, hop)
    w = torch.from_numpy(x).to(DEV)
    full = Pt.get_pitch(w)
    assert full.shape == (len(x) // hop + 1,)
    check_track(full.cpu().numpy(), PO.continuous(refw), x, fs, hop, "Pitch() continuous")
    raw = Pt.get_pitch(w, use_continuous_pitch=False).cpu().numpy()
    check_track(raw, refw, x, fs, hop, "Pitch() raw")
    F = full.numel()
    cuts = np.sort(np.random.default_rng(401).integers(0, F + 1, size=29))
    d = np.diff(np.concatenate([[0], cuts, [F]]))
    tok = Pt.get_pitch(w, use_token_averaged_pitch=True, duration=torch.from_numpy(d))
    # fp32 averages of positive values: the inputs' and each of the d - 1 sums' and the division's roundings, over the 1e-8
    rtol = (int(d.max()) + 2) * 2.0 ** -24 + REL
    np.testing.assert_allclose(tok.cpu().numpy(), PO.average_by_duration(PO.continuous(refw), d), rtol=rtol, atol=0)
    assert torch.equal(tok, align.average_by_duration(torch.from_numpy(d).float().to(DEV)[None], full[None],
                                                      torch.tensor([len(d)]), torch.tensor([full.numel()]))[0].double())


@pytest.mark.parametrize("fs", [11025, 48000])
def test_pitch_mixed_batch_is_bitwise_its_items(fs):
    hop = P.PITCH_RATE_CASES[fs][0]
    lens = [feats.pitch_min_samples(fs), fs // 2 + 3, fs, 3000, fs // 3]
    N = max(lens) + 77
    rows = np.full((len(lens), N), np.nan)
    for i, n in enumerate(lens):
        rows[i, :n] = _voice(n, fs, 500 + i, f0=110.0 + 30 * i)
    for cont, log in ((False, False), (True, True)):
        bo, bf = gpu(rows, fs, hop, continuous=cont, log=log, lengths=lens)
        for i, n in enumerate(lens):
            so, sf = gpu(rows[i, :n], fs, hop, continuous=cont, log=log)
            Fb = so.shape[1]
            assert np.array_equal(bo[i, :Fb], so[0]) and np.array_equal(bf[i, :Fb], sf[0]), (i, n)
            assert not bo[i, Fb:].any() and not bf[i, Fb:].any()
        assert (bo != 0).any()


# ---- ev_world_envelope, ev_sp2mc ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs,hop", P.WORLD_HOP_EDGES)
def test_envelope_at_the_hop_edges(lib, dev, fs, hop):
    fp = feats.pitch_frame_period(fs, hop)
    lens = [feats.pitch_min_samples(fs), int(0.2 * fs)] if hop == 16 else [int(1.5 * fs) + 5, 3 * fs]
    items = [voiced(n, fs, 600 + i) for i, n in enumerate(lens)]
    f0s = [f0_track(W.frame_count(n, fs, fp), fs, 610 + i) for i, n in enumerate(lens)]
    sp, _, st = run_envelope(lib, dev, items, fs, hop, f0s, status=True)
    assert st == 0
    worst = 0.0
    for b, it in enumerate(items):
        Fb = W.frame_count(len(it), fs, fp)
        assert (sp[b, Fb:] == 0).all()
        worst = max(worst, float(np.abs(np.log(sp[b, :Fb]) - W.cheaptrick(it, fs, f0s[b], fp, log=True)).max()))
    print("envelope fs %d hop %d: max |log sp - oracle| = %.3e (bound %.0e)" % (fs, hop, worst, LOG_BOUND))
    assert worst <= LOG_BOUND


def mc_bound(table, sp):
    """The derived bound (module docstring) per frame: table (rows, bins) host, sp (frames, bins) -> (frames, 1)."""
    rows, bins = table.shape
    s = np.abs(np.log(sp)) @ np.abs(table).T
    return (2 * (bins - 1) + bins + rows) * U * s.max(axis=1, keepdims=True)


def sp2mc_oracle(sp, order, alpha):
    """W.sp2mc of every frame at the largest order asked, sliced: freqt's c_0..c_q do not depend on the order past q."""
    return np.stack([W.sp2mc(s, order, alpha) for s in sp])


def sp2mc_gpu(lib, dev, sp, table):
    """ev_sp2mc of host sp (frames, bins) with a device table, into NaN -> host (frames, rows)."""
    x = torch.from_numpy(np.ascontiguousarray(sp)).to(dev)
    out = torch.full((sp.shape[0], table.shape[0]), math.nan, dtype=torch.float64, device=dev)
    _abi.check(lib.ev_sp2mc(x.data_ptr(), sp.shape[0], sp.shape[1], table.data_ptr(), table.shape[0], out.data_ptr(),
                            torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("fs", [8000, 16000, 48000])
def test_mel_cepstra_at_every_row_count(lib, dev, fs):
    hop = fs // 200
    fp = feats.pitch_frame_period(fs, hop)
    n_fft = W.fft_size(fs)
    items = [voiced(int(0.06 * fs), fs, 700), voiced(feats.pitch_min_samples(fs), fs, 701)]
    f0s = [f0_track(W.frame_count(len(it), fs, fp), fs, 710 + i) for i, it in enumerate(items)]
    want_sp = [W.cheaptrick(it, fs, f0s[b], fp)[:W.frame_count(len(it), fs, fp)] for b, it in enumerate(items)]
    want_all = [sp2mc_oracle(s, 255, 0.42) for s in want_sp]
    for rows in sorted(P.WORLD_ROW_CASES):
        table = feats.mcep_table(n_fft, rows - 1, 0.42, dev)
        host_table = table.cpu().numpy()
        _, mc, _ = run_envelope(lib, dev, items, fs, hop, f0s, table=table, with_sp=False)
        worst_f = worst_g = worst_ratio = 0.0
        for b, it in enumerate(items):
            Fb = want_sp[b].shape[0]
            want = want_all[b][:, :rows]
            assert (mc[b, Fb:] == 0).all()
            given = sp2mc_gpu(lib, dev, want_sp[b], table)
            ef, eg = np.abs(mc[b, :Fb] - want), np.abs(given - want)
            worst_f, worst_g = max(worst_f, float(ef.max())), max(worst_g, float(eg.max()))
            if rows > 33:
                bnd = mc_bound(host_table, want_sp[b])
                # the envelope kernel's log sp is within LOG_BOUND of the oracle's: that moves row k by sum_n |T[k, n]| LOG_BOUND
                fused = bnd + np.abs(host_table).sum(axis=1)[None, :] * LOG_BOUND
                worst_ratio = max(worst_ratio, float((ef / fused).max()), float((eg / bnd).max()))
                assert (ef <= fused).all() and (eg <= bnd).all(), (rows, float(ef.max()), float(eg.max()), float(bnd.min()))
            else:
                assert ef.max() <= MC_BOUND and eg.max() <= MC_BOUND, (rows, float(ef.max()), float(eg.max()))
        print("mel-cepstra fs %d bins %d rows %d alpha 0.42: max abs error %.3e (envelope kernel), %.3e (ev_sp2mc)%s"
              % (fs, n_fft // 2 + 1, rows, worst_f, worst_g, "; worst err / derived bound %.3g" % worst_ratio if rows > 33 else ""))


def _random_sp(frames, bins, seed):
    rng = np.random.default_rng(seed)
    return np.exp(rng.normal(-6.0, 3.0, size=(frames, bins)))


@pytest.mark.parametrize("alpha", P.WORLD_ALPHAS)
@pytest.mark.parametrize("bins", sorted(P.WORLD_BIN_CASES))
def test_sp2mc_at_every_bin_count_and_alpha(lib, dev, bins, alpha):
    n_fft = 2 * (bins - 1)
    sp = _random_sp(4, bins, bins)
    if bins > 3:                                               # an envelope's shape: the oracle's CheapTrick of a voice
        fs = {257: 8000, 513: 16000, 1025: 48000}[bins]
        x = voiced(int(0.05 * fs), fs, 800)
        fp = feats.pitch_frame_period(fs, fs // 200)
        F = W.frame_count(len(x), fs, fp)
        sp = np.concatenate([sp, W.cheaptrick(x, fs, f0_track(F, fs, 801), fp)[:4]])
    want = sp2mc_oracle(sp, 255, alpha)
    worst = {}
    for rows in (1, 25, 256):
        table = feats.mcep_table(n_fft, rows - 1, alpha, dev)
        got = sp2mc_gpu(lib, dev, sp, table)
        err = np.abs(got - want[:, :rows])
        bnd = mc_bound(table.cpu().numpy(), sp)
        if alpha == 0.42 and rows <= 33:
            bnd = np.full_like(bnd, MC_BOUND)
        worst[rows] = (float(err.max()), float((err / bnd).max()))
        assert (err <= bnd).all(), (rows, float(err.max()), float(bnd.min()))
    print("ev_sp2mc bins %d alpha %g: max abs error / worst err over bound by rows %s" % (bins, alpha, worst))


def test_sp2mc_one_frame_and_more_than_65535_frames(lib, dev):
    table = feats.mcep_table(4, 24, 0.42, dev)
    distinct = _random_sp(97, 3, 900)
    want = sp2mc_oracle(distinct, 24, 0.42)
    one = sp2mc_gpu(lib, dev, distinct[:1], table)
    assert np.abs(one - want[:1]).max() <= MC_BOUND
    n = 70001
    idx = np.arange(n) % 97
    got = sp2mc_gpu(lib, dev, distinct[idx], table)
    assert np.isfinite(got).all()
    assert np.abs(got[:97] - want).max() <= MC_BOUND
    assert got.tobytes() == got[:97][idx].tobytes()              # every row past 65535 is its twin's bits
    print("ev_sp2mc over %d frames of 3 bins: max abs error %.3e" % (n, float(np.abs(got[:97] - want).max())))


# ---- ev_eval_align -----------------------------------------------------------------------------------------------------------
def cepstra_pair(N, M, seed):
    """Cepstra (N, 24), (M, 24) and F0 tracks: the ref a time-warped noisy copy of the syn, both partly unvoiced."""
    rng = np.random.default_rng(seed)
    a = rng.normal(0.0, 0.5, size=(N, 24)) / np.arange(1, 25)
    idx = np.clip(np.round(np.linspace(0, N - 1, M) + rng.normal(0, 1.5, M)), 0, N - 1).astype(int)
    b = a[idx] + rng.normal(0, 0.02, size=(M, 24))
    fa = np.where(rng.random(N) > 0.3, rng.uniform(70, 400, N), 0.0)
    fb = np.where(rng.random(M) > 0.3, rng.uniform(70, 400, M), 0.0)
    return a, fa, b, fb


def align_call(lib, dev, pairs, extra=(3, 5)):
    """ev_eval_align on [(cep_syn, f0_syn, cep_ref, f0_ref)] with rows extra[0] / extra[1] frames past the longest item,
    NaN past each item -> [dict of stats, counts and path]."""
    B = len(pairs)
    ns, nr = [p[0].shape[0] for p in pairs], [p[2].shape[0] for p in pairs]
    max_n, max_m = max(ns), max(nr)
    Fs, Fr = max_n + extra[0], max_m + extra[1]
    cs, cr = np.full((B, Fs, 24), np.nan), np.full((B, Fr, 24), np.nan)
    fs, fr = np.full((B, Fs), np.nan), np.full((B, Fr), np.nan)
    for b, (a, fa, c, fc) in enumerate(pairs):
        cs[b, :ns[b]], fs[b, :ns[b]], cr[b, :nr[b]], fr[b, :nr[b]] = a, fa, c, fc
    t = [torch.from_numpy(x).to(dev) for x in (cs, fs, cr, fr)]
    cnt = torch.tensor(ns + nr, dtype=torch.int32, device=dev)
    stats = torch.empty((3, B), dtype=torch.float64, device=dev)
    counts = torch.empty((2, B), dtype=torch.int32, device=dev)
    stride = max_n + max_m + 1
    path = torch.full((B, stride, 2), 7, dtype=torch.int32, device=dev)
    nb = lib.ev_eval_workspace_bytes(B, max_n, max_m)
    ws = torch.full((nb,), 0xff, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_eval_align(t[0].data_ptr(), t[1].data_ptr(), Fs, cnt.data_ptr(), max_n, t[2].data_ptr(), t[3].data_ptr(), Fr,
                                 cnt.data_ptr() + 4 * B, max_m, B, stats.data_ptr(), counts.data_ptr(), path.data_ptr(), stride,
                                 ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    st, c, p = stats.cpu().numpy(), counts.cpu().numpy(), path.cpu().numpy()
    out = []
    for b in range(B):
        P_ = int(c[1, b])
        assert (p[b, P_:] == -1).all()
        out.append(dict(mcd=st[0, b], f0_rmse=st[1, b], vuv_error=st[2, b], voiced_pairs=int(c[0, b]), path_length=P_, path=p[b, :P_]))
    return out


def align_oracle(pair):
    d = O.distances(pair[0], pair[2])
    _, code = O.dtw(d)
    path = O.backtrack(code)
    want = O.statistics(d, path, pair[1], pair[3])
    want["path"] = path
    return want


def align_check(got, want, name):
    assert got["path_length"] == want["path_length"] and np.array_equal(got["path"], want["path"]), name
    assert got["voiced_pairs"] == want["voiced_pairs"], name
    worst = 0.0
    for k in ("mcd", "f0_rmse", "vuv_error"):
        r = _rel(float(got[k]), want[k])
        worst = max(worst, r)
        assert r <= 1e-12, (name, k, got[k], want[k])
    return worst


@pytest.mark.parametrize("N,M", SHAPES)
def test_eval_align_with_strides_past_the_longest_item(lib, dev, N, M):
    pair = cepstra_pair(N, M, 31 * N + M)
    got = align_call(lib, dev, [pair], extra=(3 + N % 5, 5 + M % 3))[0]
    rel = align_check(got, align_oracle(pair), (N, M))
    print("ev_eval_align N=%d M=%d: P %d, worst relative statistic error %.2e" % (N, M, got["path_length"], rel))


def test_eval_align_batch_is_bitwise_its_pairs(lib, dev):
    shapes = [(40, 60), (1, 1), (700, 650), (129, 3), (64, 64), (500, 900)]
    pairs = [cepstra_pair(n, m, 1000 + i) for i, (n, m) in enumerate(shapes)]
    batch = align_call(lib, dev, pairs, extra=(17, 1))
    rev = align_call(lib, dev, pairs[::-1], extra=(1, 29))[::-1]
    for b, pair in enumerate(pairs):
        alone = align_call(lib, dev, [pair], extra=(0, 0))[0]
        align_check(alone, align_oracle(pair), shapes[b])
        for other in (batch[b], rev[b]):
            for k in ("mcd", "f0_rmse", "vuv_error", "voiced_pairs", "path_length"):
                assert np.asarray(other[k]).tobytes() == np.asarray(alone[k]).tobytes(), (b, k)
            assert np.array_equal(other["path"], alone["path"]), b
