"""Loudness normalisation on the host (no GPU): the K-weighting coefficients against BS.1770-4's table, the fp64 oracle's known
answers, the per-sub-block restart ev_loudness uses against sequential filtering, torchaudio's independent meter, the target
checks, and the MicroBatcher's format keys."""
import numpy as np
import pytest
import torch
from scipy.signal import freqz, lfilter

from conftest import load_golden
from emotivoice_b200 import audio
from emotivoice_b200 import frontdoor as fd
from oracle import loudness_oracle as O

SR = 16000


def _flat(sb, sa, hb, ha):
    return np.concatenate([sb, sa[1:], hb, ha[1:]])


def _table():
    t = O.TABLE_48K
    return np.array(t["shelf_b"] + t["shelf_a"][1:] + t["hp_b"] + t["hp_a"][1:])


def test_k_weighting_is_the_standards_table_at_48k_and_both_agree_at_16k():
    assert np.abs(audio.k_weighting(48000) - _table()).max() <= 1e-12
    assert np.abs(_flat(*O.k_weighting(48000)) - _table()).max() <= 1e-12
    k16 = audio.k_weighting(SR)
    assert k16.dtype == np.float64 and k16.shape == (10,)
    assert np.abs(k16 - _flat(*O.k_weighting(SR))).max() <= 1e-12


def _k_gain_db(f):
    sb, sa, hb, ha = O.k_weighting(SR)
    w = 2 * np.pi * f / SR
    return 20 * np.log10(abs(freqz(sb, sa, [w])[1][0] * freqz(hb, ha, [w])[1][0]))


def _sine(dbfs, seconds, f=1000.0):
    n = np.arange(int(round(seconds * SR)))
    return 10.0 ** (dbfs / 20.0) * np.sin(2 * np.pi * f * n / SR)


@pytest.mark.parametrize("amp", [1.0, 0.5, 0.01])
def test_sine_reads_its_power_plus_the_k_weight(amp):
    assert abs(_k_gain_db(997.0) - 0.731) < 1e-3
    x = amp * np.sin(2 * np.pi * 997.0 * np.arange(20 * SR) / SR)
    want = 20 * np.log10(amp) - 3.0103 + (_k_gain_db(997.0) - 0.691)
    assert abs(O.integrated_loudness(x, SR) - want) <= 1e-3


def _case5():
    """EBU Tech 3341 case 5 in mono: -36 / -23 / -36 dBFS 1 kHz sine for 10 / 60 / 10 s."""
    return np.concatenate([_sine(-36, 10), _sine(-23, 60), _sine(-36, 10)])


def test_tech3341_case5_reads_the_loud_part():
    L = O.integrated_loudness(_case5(), SR)
    assert abs(L - O.integrated_loudness(_sine(-23, 60), SR)) <= 0.05
    assert abs(L - (-25.99)) <= 0.01


def test_blocks_below_the_absolute_gate_are_ignored():
    loud = _sine(-20, 10)
    quiet = 10.0 ** (-80 / 20) * np.random.default_rng(1).standard_normal(10 * SR)
    L, l, _ = O.gating(np.concatenate([loud, quiet]), SR)
    # the blocks that hold a loud sub-block are those of loud + 300 ms of quiet.  The next one holds the filters' ringing and
    # passes the absolute gate but not the relative one; every later block is below -70 LUFS
    head = np.concatenate([loud, quiet[:3 * SR // 10]])
    z = O.block_mean_squares(head, SR)
    assert len(z) == 100 and np.all(l[:100] > -40) and -70 < l[100] < -40 and np.all(l[101:] < -70)
    assert abs(L - (-0.691 + 10 * np.log10(z.mean()))) <= 1e-9
    assert O.integrated_loudness(_sine(-75, 5), SR) == -np.inf


def test_short_and_silent_inputs_read_minus_infinity():
    x = np.random.default_rng(2).uniform(-0.5, 0.5, 6401)
    assert O.integrated_loudness(x[:6399], SR) == -np.inf
    assert len(O.block_mean_squares(x[:6400], SR)) == 1
    assert np.isfinite(O.integrated_loudness(x[:6400], SR))
    assert O.integrated_loudness(np.zeros(5 * SR), SR) == -np.inf
    assert O.gain(-np.inf, 0.0, -23.0) == 1.0


def _restart_energies(x, kc, W):
    """Sub-block sums of squares as ev_loudness forms them: each 100 ms sub-block filtered from zero state W samples before it."""
    S = SR // 10
    sb, sa, hb, ha = kc[0:3], np.r_[1.0, kc[3:5]], kc[5:8], np.r_[1.0, kc[8:10]]
    out = []
    for j in range(len(x) // S):
        s0 = max(0, j * S - W)
        y = lfilter(hb, ha, lfilter(sb, sa, x[s0:(j + 1) * S]))[-S:]
        out.append(np.sum(y * y))
    return np.array(out)


@pytest.mark.parametrize("name", ["noise", "dc_step", "b1_t100"])
def test_sub_block_restart_matches_sequential_filtering(name):
    rng = np.random.default_rng(3)
    if name == "noise":
        x = rng.uniform(-1.0, 1.0, 12 * SR)
    elif name == "dc_step":
        x = np.zeros(8 * SR)
        x[3 * SR + 123:] = 0.9
    else:
        x = load_golden("b1_t100")["wav"][0, 0].double().numpy()
    kc = audio.k_weighting(SR)
    W = audio.restart_warmup(kc)
    assert W == 2048
    S = SR // 10
    y = O.k_filter(x, SR)
    seq = np.sum((y[:len(x) // S * S] ** 2).reshape(-1, S), axis=1)
    got = _restart_energies(x, kc, W)
    # relative to the sub-block's energy, or to a sub-block at the absolute gate's level (-70 LUFS) where it is quieter: below
    # that a block never enters the result
    floor = S * 10.0 ** ((-70 + 0.691) / 10)
    err = np.abs(got - seq) / np.maximum(seq, floor)
    assert err.max() <= 1e-9, err.max()


def test_torchaudio_meter_agrees_on_case5():
    import torchaudio.functional as F
    x = _case5()
    ta = float(F.loudness(torch.from_numpy(x)[None].float(), SR))
    assert abs(ta - O.integrated_loudness(x, SR)) <= 0.2


def test_loudness_targets_are_checked():
    assert audio.check_loudness(-23) == -23.0 and audio.check_loudness(np.float32(-16.0)) == -16.0
    assert audio.check_loudness(0) == 0.0 and audio.check_loudness(-70.0) == -70.0
    for bad in (float("nan"), float("inf"), -float("inf"), 0.5, -70.01, -100, True, False, "-23", None, [-23]):
        with pytest.raises(ValueError):
            audio.check_loudness(bad)


def test_microbatcher_measures_and_formats_once_per_key(monkeypatch):
    wav = torch.zeros(5, 1, 512)

    def forward(**kw):
        return {"wav_predictions": wav[:len(kw["inputs_ling"])], "mel_lengths": torch.full((len(kw["inputs_ling"]),), 2)}

    calls = []

    def fake_fetch(model, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None):
        calls.append((sample_rate, encoding, loudness, true_peak, tuple(items)))
        return [np.array([sample_rate or 0, len(calls)]) for _ in items]

    monkeypatch.setattr(fd, "fetch_audio", fake_fetch)
    z = np.zeros(768, np.float32)
    reqs = [dict(loudness=-23), dict(loudness=-16, encoding="mulaw", sample_rate=8000), dict(loudness=-23.0),
            dict(loudness=-23, sample_rate=24000), dict()]
    with fd.MicroBatcher(forward, max_batch=5, max_wait_s=0.5) as mb:
        for kw in (dict(loudness=float("nan")), dict(loudness=3.0), dict(loudness="loud"), dict(loudness=True)):
            with pytest.raises(ValueError):
                mb.submit(np.array([1, 2]), 0, z, z, **kw)
            with pytest.raises(ValueError):
                mb.submit_joined([np.array([1, 2])], 0, z, z, **kw)
        futs = [mb.submit(np.array([1, 2, 3]), 0, z, z, **kw) for kw in reqs]
        got = [f.result(timeout=30) for f in futs]
        assert mb.batches_run == 1
    assert sorted(calls, key=str) == sorted([(16000, "pcm16", -23.0, None, (0, 2)), (8000, "mulaw", -16.0, None, (1,)),
                                             (24000, "pcm16", -23.0, None, (3,))], key=str)
    assert isinstance(got[4], torch.Tensor)
    assert got[0][1] == got[2][1]                   # one call served both -23 LUFS requests at 16 kHz PCM16
    assert fd.MicroBatcher._output_format(mb, None, None, -23) == audio.OutputFormat(16000, 1, 1, "pcm16", -23.0, None)
    assert fd.MicroBatcher._output_format(mb, None, None, None) is None
    assert fd.MicroBatcher._output_format(mb, None, "alaw", None) == audio.OutputFormat(16000, 1, 1, "alaw", None, None)
