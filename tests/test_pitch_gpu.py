"""ev_pitch (csrc/pitch_kernels.cu) through emotivoice_b200.feats.Pitch against the fp64 restatement of pyworld.dio /
pyworld.stonemask (oracle/pitch_oracle.py): every fixture, length edges, a 30 s item, batches, silence and one chain from a
recording into the model's forward(pitch=).

Bound: 1e-8 relative on every voiced frame, with the voiced/unvoiced masks identical.  The kernels compute each band signal by
direct fp64 FIR in the oracle's tap order, but their taps come from the device's cos (within 2 ulp of libm's), and StoneMask's
DFT sums run in a warp-tree order: each band sample differs from the oracle's by at most ~2600 taps x 2^-52 of the sum of its
|terms|, about 1e-13 relative.  An event's fine position moves by that over the band signal's slope, below 1e-10 samples on
these signals, and an F0 of fs / (>= 20 samples) by under 1e-11 relative; StoneMask's bins over <= 3601 samples add about
1e-13.  1e-8 leaves three orders of headroom over that sum; a flipped decision (a zero-crossing sign, an argmin, an
allowed_range test) shows up as a mask difference or an error of percents, far above it.  Token averages go through the fp32
ev_op_average_by_duration: they are checked to fp32 rounding (2^-22 relative) and bit for bit against align.average_by_duration.
"""
import glob
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from emotivoice_b200 import align, feats, synth
from oracle import pitch_oracle as PO

pytestmark = pytest.mark.gpu
DEV = "cuda"
REL = 1e-8
FIXTURES = sorted(os.path.basename(p)[6:-4] for p in glob.glob(os.path.join(GOLDEN, "pitch_*.npz")))
KNOWN = ["stat90", "stat150", "stat220", "stat330", "vibrato", "glide", "sr24k"]


def load(name):
    with np.load(os.path.join(GOLDEN, "pitch_%s.npz" % name)) as z:
        return {k: z[k] for k in z.files}


def gpu(x, sr, hop, continuous=False, log=False, lengths=None):
    t = torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    out, f0 = feats.pitch_track(t if t.dim() == 2 else t[None], sr, hop, continuous, log, lengths, raw=True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), f0.cpu().numpy()


def _evidence(x, sr, hop, frames):
    _, _, det = PO.dio(np.asarray(x, np.float64), sr, 1000 * hop / sr, details=True)
    rows = []
    for f in frames[:4]:
        rows.append("frame %d: best %.12g, candidates %s, scores %s" % (f, det["best"][f], np.array2string(det["candidates"][:, f], precision=9),
                                                                         np.array2string(det["scores"][:, f], precision=6)))
    return "\n".join(rows)


def check_track(got, want, x, sr, hop, what):
    m_got, m_want = got != 0, want != 0
    bad = np.nonzero(m_got != m_want)[0]
    assert bad.size == 0, "%s: voicing differs at frames %s (gpu %s, oracle %s)\n%s" % (
        what, bad[:8], got[bad[:8]], want[bad[:8]], _evidence(x, sr, hop, bad))
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-300)
    rel[~m_want] = 0
    worst = np.nonzero(rel > REL)[0]
    assert worst.size == 0, "%s: rel error %.3e > %g at frames %s (gpu %s, oracle %s)\n%s" % (
        what, rel.max(), REL, worst[:8], got[worst[:8]], want[worst[:8]], _evidence(x, sr, hop, worst))


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name):
    z = load(name)
    sr, hop = int(z["sr"]), int(z["hop"])
    for inp in (z["wav"], z["wav"].astype(np.float64)):
        ref, f0 = gpu(inp, sr, hop)
        check_track(f0[0], z["f0_dio"], z["wav"], sr, hop, "dio")
        check_track(ref[0], z["f0_refined"], z["wav"], sr, hop, "refined")
    cont, _ = gpu(z["wav"], sr, hop, continuous=True)
    check_track(cont[0], z["continuous"], z["wav"], sr, hop, "continuous")
    lg, _ = gpu(z["wav"], sr, hop, continuous=True, log=True)
    check_track(lg[0], z["log"], z["wav"], sr, hop, "log")
    lr, _ = gpu(z["wav"], sr, hop, continuous=False, log=True)
    check_track(lr[0], z["log_raw"], z["wav"], sr, hop, "log without interpolation")
    P = feats.Pitch(sr=sr, hop_length=hop)
    w = torch.from_numpy(z["wav"]).to(DEV)
    tok = P.get_pitch(w, use_token_averaged_pitch=True, duration=torch.from_numpy(z["durations"]))
    assert tok.dtype == torch.float64 and tok.shape == z["token_avg"].shape
    np.testing.assert_allclose(tok.cpu().numpy(), z["token_avg"], rtol=2.0 ** -22, atol=0)
    full = P.get_pitch(w)
    assert full.dtype == torch.float64 and full.shape == (len(z["wav"]) // hop + 1,)
    assert torch.equal(tok, align.average_by_duration(torch.from_numpy(z["durations"]).float().to(DEV)[None], full[None],
                                                      torch.tensor([len(z["durations"])]), torch.tensor([full.numel()]))[0].double())


def _voice(n, sr, seed, f0=180.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    ph = 2 * np.pi * np.cumsum(f0 * (1 + 0.04 * np.sin(2 * np.pi * 5 * t))) / sr
    return sum(0.3 / k * np.sin(k * ph + k) for k in range(1, 6)) + 1e-4 * rng.standard_normal(n)


def _oracle_all(x, sr, hop):
    f0, t = PO.dio(x, sr, 1000 * hop / sr)
    ref = PO.stonemask(x, f0, t, sr)
    return f0, ref


@pytest.mark.parametrize("n", [641, 642, 767, 768, 769, 4 * 256 - 1, 4 * 256, 4 * 256 + 1, 40 * 256 - 1, 40 * 256, 40 * 256 + 1])
def test_length_edges(n):
    x = _voice(n, 16000, n)
    f0w, refw = _oracle_all(x, 16000, 256)
    ref, f0 = gpu(x, 16000, 256)
    assert f0.shape == (1, n // 256 + 1)
    check_track(f0[0], f0w, x, 16000, 256, "dio n=%d" % n)
    check_track(ref[0], refw, x, 16000, 256, "refined n=%d" % n)


@pytest.mark.parametrize("sr,hop", [(22050, 256), (48000, 300)])
def test_other_rates(sr, hop):
    x = _voice(int(1.2 * sr), sr, sr, f0=140.0)
    f0w, refw = _oracle_all(x, sr, hop)
    ref, f0 = gpu(x, sr, hop)
    check_track(f0[0], f0w, x, sr, hop, "dio %d" % sr)
    check_track(ref[0], refw, x, sr, hop, "refined %d" % sr)
    assert (refw > 0).sum() > 0.8 * len(refw)


def test_thirty_seconds():
    x = _voice(30 * 16000, 16000, 30)
    f0w, refw = _oracle_all(x, 16000, 256)
    ref, f0 = gpu(x, 16000, 256)
    check_track(f0[0], f0w, x, 16000, 256, "dio 30 s")
    check_track(ref[0], refw, x, 16000, 256, "refined 30 s")


def test_shortest_item_and_too_short():
    n = feats.pitch_min_samples(16000)
    x = torch.from_numpy(_voice(n, 16000, 1)).to(DEV)
    out = feats.Pitch(sr=16000, hop_length=256).get_pitch(x)
    assert out.shape == (n // 256 + 1,) and not out.any()          # 3 frames: FixF0Contour leaves them 0
    with pytest.raises(ValueError):
        feats.Pitch(sr=16000, hop_length=256).get_pitch(x[:n - 1])
    with pytest.raises(ValueError):
        feats.pitch_track(torch.zeros(2, 4000, device=DEV), 16000, 256, lengths=[4000, 640])
    with pytest.raises(ValueError):
        feats.pitch_track(torch.zeros(2, 4000, device=DEV), 16000, 256, lengths=[4000])
    with pytest.raises(ValueError):
        feats.pitch_track(torch.zeros(2, 4000, device=DEV), 16000, 256, lengths=[4000, 4001])
    with pytest.raises(ValueError):
        feats.Pitch(sr=16000, hop_length=256).get_pitch(torch.zeros(2, 4000, device=DEV), use_token_averaged_pitch=True, duration=[1])


@pytest.mark.parametrize("name", KNOWN)
def test_known_f0_on_gpu(name):
    from test_pitch import core_frames
    z = load(name)
    sr, hop = int(z["sr"]), int(z["hop"])
    ref, _ = gpu(z["wav"], sr, hop)
    core = core_frames(z["known_f0"])
    assert (ref[0][core] > 0).all()
    assert np.abs(ref[0][core] / z["known_f0"][core] - 1).max() <= 0.01


def test_batch_is_bitwise_single_calls():
    lens = [16000, 9001, 4097, 12800]
    N = max(lens)
    rows = np.full((len(lens), N), np.nan)
    for i, n in enumerate(lens):
        rows[i, :n] = _voice(n, 16000, 100 + i, f0=120.0 + 40 * i)
    for cont, log in ((False, False), (True, True)):
        bo, bf = gpu(rows, 16000, 256, continuous=cont, log=log, lengths=lens)
        F = N // 256 + 1
        assert bo.shape == (len(lens), F)
        for i, n in enumerate(lens):
            so, sf = gpu(rows[i, :n], 16000, 256, continuous=cont, log=log)
            Fb = n // 256 + 1
            assert np.array_equal(bo[i, :Fb], so[0]) and np.array_equal(bf[i, :Fb], sf[0])
            assert not bo[i, Fb:].any() and not bf[i, Fb:].any()
        assert (bo[:, :10] != 0).any()


def test_digital_silence():
    P = feats.Pitch(sr=16000, hop_length=256)
    for dt in (torch.float32, torch.float64):
        z = torch.zeros(2, 20000, dtype=dt, device=DEV)
        for cont in (True, False):
            out = P.get_pitch(z, use_continuous_pitch=cont, use_log_pitch=True)
            assert out.dtype == torch.float64 and out.shape == (2, 20000 // 256 + 1) and not out.any()


def test_chain_into_forward(model, dev):
    """b1_t100's waveform -> Pitch frames == TacotronSTFT frames -> token averages over viterbi_decode durations ->
    pitch_stats normalisation -> forward(pitch=)."""
    from conftest import load_golden
    g = load_golden("b1_t100")
    wav = g["wav"].reshape(-1).to(DEV)
    mel = feats.TacotronSTFT(sampling_rate=16000).to(DEV).mel_spectrogram(wav[None])
    F = mel.shape[-1]
    P = feats.Pitch(sr=16000, hop_length=256)
    frames = P.get_pitch(wav)
    assert frames.shape == (F,)
    adim, odim, T = 384, 80, 40
    mod = align.AlignmentModule(adim, odim)
    mod.load_state_dict(synth.make_alignment_state_dict(adim, odim))
    mod = mod.to(DEV)
    text = torch.from_numpy(np.random.default_rng(9500).normal(size=(1, T, adim)).astype(np.float32)).to(DEV)
    tl, fl = torch.tensor([T]), torch.tensor([F])
    ds, _ = align.viterbi_decode(mod(text, mel.transpose(1, 2), tl, fl), tl, fl)
    tok = P.get_pitch(wav, use_token_averaged_pitch=True, duration=ds[0])
    assert torch.equal(tok, align.average_by_duration(ds, frames[None], tl, fl)[0].double())
    norm = (tok - 225.089) / 53.78
    Tm = g["inputs_ling"].shape[1]
    track = norm.float().repeat((Tm + T - 1) // T)[:Tm][None]
    keys = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
    plain = model(**{k: g[k].to(dev) for k in keys})
    fed = model(**{k: g[k].to(dev) for k in keys}, pitch=track.to(dev))
    torch.cuda.synchronize()
    assert torch.equal(plain["mel_lengths"], fed["mel_lengths"])
    assert torch.isfinite(fed["wav_predictions"]).all()
