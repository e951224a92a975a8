"""Prosody controls (duration_scale / pitch_shift / energy_scale) without a GPU: the oracle against the fixtures that
oracle/make_golden_prosody.py generated from the unmodified reference, host validation and packing, the front door's
per-item controls, and the new C symbols."""
import math
import threading

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max
from emotivoice_b200 import frontdoor as fd
from emotivoice_b200 import _abi
from emotivoice_b200.modules import prosody_table
from oracle import prosody_oracle as O

KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
CONTROLS = ("duration_scale", "pitch_shift", "energy_scale")
ITEM_CASES = ["a050", "a080", "a125", "a200", "p_up4", "p_down4", "e070", "e130", "combined", "mixed3", "zero_dur"]


def controls_of(g):
    return {c: g[c].tolist() for c in CONTROLS}


def state_dict_for(sd, g):
    if "dur_bias" not in g:
        return sd
    out = dict(sd)
    out["am.duration_predictor.linear.bias"] = torch.full_like(sd["am.duration_predictor.linear.bias"], float(g["dur_bias"]))
    return out


@pytest.mark.parametrize("name", ITEM_CASES)
def test_oracle_reproduces_per_item_prosody_fixture(name, sd, conf):
    g = load_golden("prosody_" + name)
    per = O.jets_forward_per_utterance(state_dict_for(sd, g), conf, {k: g[k] for k in KEYS}, controls=controls_of(g))
    for b, o in enumerate(per):
        assert torch.equal(o["log_duration_predictions"], g["durations_%d" % b])
        assert torch.equal(o["mel_lens"], g["mel_lens_%d" % b])
        assert o["dec_outputs"].shape == g["mel_%d" % b].shape
        assert rel_max(o["dec_outputs"], g["mel_%d" % b]) <= 2e-6
        assert rel_max(o["wav_predictions"], g["wav_%d" % b]) <= 2e-6
        assert rel_max(o["pitch_predictions"].reshape(1, -1), g["pitch_%d" % b]) <= 2e-6    # raw predictions, not shifted


def test_oracle_reproduces_padded_prosody_fixture(sd, conf):
    g = load_golden("prosody_padded")
    assert bool(g["literal"])
    o = O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, **controls_of(g))
    assert torch.equal(o["log_duration_predictions"], g["durations"])
    assert torch.equal(o["mel_lens"], g["mel_lens"])
    assert rel_max(o["dec_outputs"], g["mel"]) <= 2e-6
    assert rel_max(o["wav_predictions"], g["wav"]) <= 2e-6


def test_rate_fixtures_scale_the_frame_count(sd, conf):
    """ds = fl32(d * alpha): alpha = 0.5 and 2 are exact, so their frame counts follow from the neutral one."""
    assert int(load_golden("prosody_a200")["mel_lens_0"][0]) == 2 * int(load_golden("b1_t50")["mel"].shape[1])
    base = int(load_golden("b1_t100")["mel"].shape[1])
    assert int(load_golden("prosody_a050")["mel_lens_0"][0]) == base // 2
    d = load_golden("prosody_a080")["durations_0"]
    assert int(load_golden("prosody_a080")["mel_lens_0"][0]) == int(np.float32((d.float() * 0.8).double().sum().item()))


def test_neutral_prosody_oracle_is_the_jets_oracle(sd, conf):
    """The restatement with controls computes exactly what oracle/jets_oracle.py computes when they are neutral."""
    from oracle import jets_oracle as J
    g = load_golden("b3_padded")
    batch = {k: g[k] for k in KEYS}
    want = J.jets_forward(sd, conf, **batch)
    for kw in ({}, dict(duration_scale=[1.0] * 3, pitch_shift=0.0, energy_scale=1.0)):
        got = O.jets_forward(sd, conf, **batch, **kw)
        for k in ("dec_outputs", "wav_predictions", "log_duration_predictions", "pitch_predictions", "mel_lens"):
            assert torch.equal(got[k], want[k]), k
    # the same through the controlled path: an explicit neutral table (p * 1 + 0, ds * 1.0) changes no bit
    m = O.acoustic_model(sd, conf, *(batch[k] for k in KEYS), prosody=torch.tensor([[1.0, 1.0, 0.0, 1.0, 0.0]] * 3))
    assert torch.equal(m["dec_outputs"], want["dec_outputs"]) and torch.equal(m["mel_lens"], want["mel_lens"])


def test_zero_duration_guard_writes_one_not_alpha(sd, conf):
    g = load_golden("prosody_zero_dur")
    assert int(g["durations_0"].abs().sum()) == 0 and g["duration_scale"].tolist() == [0.75]
    assert int(g["mel_lens_0"][0]) == int(g["input_lengths"][0])          # every token got 1 frame


def test_zero_frame_fixture_is_a_reference_error(sd, conf):
    """Scaled to zero frames the reference raises RuntimeError in the decoder; so does the oracle."""
    g = load_golden("prosody_zero_frames")
    assert bool(g["reference_raises"])
    with pytest.raises(RuntimeError):
        O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, **controls_of(g))


# ---- host validation and packing -------------------------------------------------------------------------------------

def test_prosody_table_neutral_is_none_and_matches_the_oracle(conf):
    assert prosody_table(3) is None
    assert prosody_table(2, 1.0, 0.0, 1.0) is None
    assert prosody_table(2, [1.0, 1.0], torch.zeros(2), np.ones(2)) is None
    kw = dict(duration_scale=[0.8, 1.0, 1 / 1.3], pitch_shift=[4.0, 0.0, -2.5], energy_scale=[1.0, 1.3, 0.7])
    t = prosody_table(3, config=conf, **kw)
    assert t.dtype == torch.float32 and t.shape == (3, 5) and t.device.type == "cpu"
    assert torch.equal(t, O.prosody_table(3, **kw))
    assert t[1].tolist() == [1.0, 1.0, 0.0, np.float32(1.3), np.float32(30.610 * 0.3 / 21.78)]
    r = 2.0 ** (4 / 12)
    assert t[0, 1].item() == np.float32(r) and t[0, 2].item() == np.float32(225.089 * (r - 1) / 53.78)
    assert torch.equal(prosody_table(3, 0.5), torch.tensor([[0.5, 1, 0, 1, 0]] * 3, dtype=torch.float32))


def test_prosody_table_uses_the_config_statistics(conf):
    from emotivoice_b200.config import AttrDict
    c = AttrDict(conf)
    c["pitch_stats"] = [200.0, 50.0]
    c["energy_stats"] = [30.0, 20.0]
    t = prosody_table(1, pitch_shift=12.0, energy_scale=2.0, config=c)
    assert t[0].tolist() == [1.0, 2.0, 4.0, 2.0, 1.5]


@pytest.mark.parametrize("kw", [
    dict(duration_scale=0.0), dict(duration_scale=-1.0), dict(duration_scale=math.inf), dict(duration_scale=math.nan),
    dict(duration_scale=[1.0, 0.0]), dict(energy_scale=0.0), dict(energy_scale=-0.5), dict(energy_scale=math.inf),
    dict(pitch_shift=math.nan), dict(pitch_shift=[0.0, -math.inf]), dict(pitch_shift=1e6),
    dict(duration_scale=[1.0, 2.0, 3.0]), dict(pitch_shift=[1.0]), dict(energy_scale=torch.ones(3)),
    dict(duration_scale=1e-50), dict(duration_scale=1e50), dict(duration_scale="fast"),
], ids=lambda kw: "%s=%r" % next(iter(kw.items())))
def test_prosody_table_rejects_bad_values(kw):
    with pytest.raises(ValueError):
        prosody_table(2, **kw)


def test_prosody_table_rejects_device_tensors():
    with pytest.raises(ValueError, match="CPU tensor"):
        prosody_table(2, duration_scale=torch.ones(2, device="meta"))


def test_forward_validates_before_touching_the_engine(conf):
    """A bad control raises ValueError even where there is no GPU: nothing is packed or enqueued first."""
    from emotivoice_b200 import synth
    from emotivoice_b200.modules import JETSGenerator
    m = JETSGenerator(conf)
    batch = synth.make_batch([5, 7])
    for kw in (dict(duration_scale=0.0), dict(pitch_shift=math.nan), dict(energy_scale=[1.0]),
               dict(duration_scale=torch.ones(2, device="meta"))):
        with pytest.raises(ValueError):
            m(**batch, **kw)
        with pytest.raises(ValueError):
            m.am(**batch, **kw)
    assert m._ev_engine is None
    with pytest.raises(RuntimeError, match="no CPU fallback"):        # valid controls reach the engine as usual
        m(**batch, duration_scale=[1.0, 0.8], alpha=3.0)


def test_new_symbols_are_declared():
    for name in ("ev_am_phase1_prosody", "ev_op_duration_scan"):
        assert name in _abi.SIGNATURES


# ---- front door ------------------------------------------------------------------------------------------------------

def test_speech_controls_map_speed_to_duration_scale():
    assert fd.speech_controls() == fd.NEUTRAL_CONTROLS
    assert fd.speech_controls(speed=1.25, pitch_shift=2, energy_scale=0.5) == (1 / 1.25, 2.0, 0.5)
    for kw in (dict(speed=0), dict(speed=-2.0), dict(speed=math.inf), dict(pitch_shift=math.nan), dict(energy_scale=0.0)):
        with pytest.raises(ValueError):
            fd.speech_controls(**kw)


def test_collate_carries_controls_only_when_some_item_is_not_neutral():
    z = np.zeros(8, np.float32)
    neutral = [(np.array([1, 2]), 0, z, z), (np.array([3]), 1, z, z, fd.NEUTRAL_CONTROLS)]
    assert set(fd.collate(neutral)) == set(KEYS)
    mixed = neutral + [(np.array([4, 5, 6]), 2, z, z, fd.speech_controls(speed=2.0, pitch_shift=-3.0))]
    b = fd.collate(mixed)
    assert b["duration_scale"] == [1.0, 1.0, 0.5]
    assert b["pitch_shift"] == [0.0, 0.0, -3.0] and b["energy_scale"] == [1.0, 1.0, 1.0]
    assert b["inputs_ling"].shape == (3, 3)


def _fake_model(calls):
    """2 frames per phoneme times duration_scale (truncated), the sample value encodes the item's pitch shift."""
    def forward(inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding, **controls):
        calls.append(controls)
        B = inputs_ling.shape[0]
        ds = controls.get("duration_scale", [1.0] * B)
        ps = controls.get("pitch_shift", [0.0] * B)
        mel = torch.tensor([int(2 * int(input_lengths[b]) * ds[b]) for b in range(B)], dtype=torch.int32)
        wav = torch.zeros(B, 1, int(mel.max()) * 256)
        for b in range(B):
            wav[b, 0, :int(mel[b]) * 256] = float(inputs_speaker[b]) + ps[b]
        return {"wav_predictions": wav, "mel_lengths": mel}
    return forward


def test_microbatcher_shares_one_forward_between_different_controls():
    calls = []
    z = np.zeros(8, np.float32)
    reqs = [dict(speed=1.0), dict(speed=2.0, pitch_shift=3.0), dict(speed=0.5, energy_scale=1.2), dict()]
    with fd.MicroBatcher(_fake_model(calls), max_batch=4, max_wait_s=0.5) as mb:
        barrier = threading.Barrier(len(reqs))
        futs = [None] * len(reqs)

        def worker(i):
            barrier.wait()
            futs[i] = mb.submit(np.arange(1, 11), i, z, z, **reqs[i])

        ths = [threading.Thread(target=worker, args=(i,)) for i in range(len(reqs))]
        [t.start() for t in ths]
        [t.join() for t in ths]
        outs = [f.result(timeout=10) for f in futs]
        with pytest.raises(ValueError):
            mb.submit(np.arange(3), 0, z, z, speed=0.0)                 # rejected at submit, never reaches a batch
    assert len(calls) == 1 and sorted(calls[0]) == sorted(CONTROLS)
    frames = [20, 10, 40, 20]
    for i, w in enumerate(outs):
        assert w.shape == (frames[i] * 256,)
        assert torch.all(w == i + reqs[i].get("pitch_shift", 0.0))


def test_microbatcher_neutral_traffic_makes_the_plain_call():
    calls = []
    z = np.zeros(8, np.float32)
    with fd.MicroBatcher(_fake_model(calls), max_batch=2, max_wait_s=0.01) as mb:
        assert mb.submit(np.arange(1, 4), 0, z, z, speed=1.0).result(timeout=10).shape == (6 * 256,)
    assert calls == [{}]
