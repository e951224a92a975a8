"""Phoneme-level prosody controls and caller-given durations / pitch / energy without a GPU: the oracle against the fixtures
that oracle/make_golden_token_prosody.py generated from the unmodified reference, host validation of the (B,T) controls and
caller values (raising before anything is enqueued), the front door's padding, and the new C symbols."""
import math
import threading

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max
from emotivoice_b200 import frontdoor as fd
from emotivoice_b200 import _abi, synth
from emotivoice_b200.modules import JETSGenerator, caller_values, prosody_table
from oracle import prosody_oracle as P
from oracle import token_prosody_oracle as O

KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
EXTRA = ("duration_scale", "pitch_shift", "energy_scale", "durations", "pitch", "energy")
ITEM_CASES = ["pause_word", "pitch_span", "caller_dur", "caller_pe", "mixed3"]


def extras_of(g):
    return {k: g[k].numpy() for k in EXTRA if k in g}


# ---- the oracle against the reference fixtures ------------------------------------------------------------------------

@pytest.mark.parametrize("name", ITEM_CASES)
def test_oracle_reproduces_token_prosody_fixture(name, sd, conf):
    g = load_golden("token_prosody_" + name)
    assert not bool(g["literal"])
    per = O.jets_forward_per_utterance(sd, conf, {k: g[k] for k in KEYS}, controls=extras_of(g))
    for b, o in enumerate(per):
        assert torch.equal(o["log_duration_predictions"], g["pred_durations_%d" % b])
        assert torch.equal(o["mel_lens"], g["mel_lens_%d" % b])
        assert o["dec_outputs"].shape == g["mel_%d" % b].shape
        assert rel_max(o["dec_outputs"], g["mel_%d" % b]) <= 2e-6
        assert rel_max(o["wav_predictions"], g["wav_%d" % b]) <= 2e-6
        assert rel_max(o["pitch_predictions"].reshape(1, -1), g["pred_pitch_%d" % b]) <= 2e-6     # raw predictions


def test_oracle_reproduces_padded_token_prosody_fixture(sd, conf):
    g = load_golden("token_prosody_padded")
    assert bool(g["literal"])
    o = O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, **extras_of(g))
    assert torch.equal(o["log_duration_predictions"], g["pred_durations"])
    assert torch.equal(o["mel_lens"], g["mel_lens"])
    assert rel_max(o["dec_outputs"], g["mel"]) <= 2e-6
    assert rel_max(o["wav_predictions"], g["wav"]) <= 2e-6


def test_caller_duration_fixture_counts_the_given_frames():
    """Item 0: the caller's durations (pads ignored) times 1.3; item 1: all zero, the guard gives each phoneme one frame."""
    g = load_golden("token_prosody_caller_dur")
    d, n0, n1 = g["durations"], int(g["input_lengths"][0]), int(g["input_lengths"][1])
    assert int(g["mel_lens_0"][0]) == int(np.float32((d[0, :n0].float() * np.float32(1.3)).double().sum().item()))
    assert int(d[1].abs().sum()) == 0 and int(g["mel_lens_1"][0]) == n1
    assert int(d[0, n0:].abs().sum()) > 0                  # garbage past the item's length, which the model ignores


def test_zero_frame_fixture_is_a_reference_error(sd, conf):
    g = load_golden("token_prosody_zero_frames")
    assert bool(g["reference_raises"])
    with pytest.raises(RuntimeError):
        O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, **extras_of(g))


def test_token_oracle_with_constant_rows_is_the_per_item_oracle(sd, conf):
    """A (B,T) table whose rows repeat one value computes exactly what the per-item oracle computes; so does feeding the
    predictions back as caller values."""
    g = load_golden("prosody_mixed3")
    batch = {k: g[k] for k in KEYS}
    c = {k: g[k].tolist() for k in ("duration_scale", "pitch_shift", "energy_scale")}
    T = int(batch["inputs_ling"].shape[1])
    want = P.jets_forward_per_utterance(sd, conf, batch, controls=c)
    rows = {k: np.repeat(np.asarray(v, dtype=np.float64)[:, None], T, axis=1) for k, v in c.items()}
    got = O.jets_forward_per_utterance(sd, conf, batch, controls=rows)
    for w, o in zip(want, got):
        for k in ("dec_outputs", "wav_predictions", "log_duration_predictions", "mel_lens"):
            assert torch.equal(w[k], o[k]), k
    one = synth.slice_batch(batch, 1)
    plain = O.jets_forward(sd, conf, **one)
    fed = O.jets_forward(sd, conf, **one, durations=plain["log_duration_predictions"], pitch=plain["pitch_predictions"],
                         energy=plain["energy_predictions"])
    for k in ("dec_outputs", "wav_predictions", "mel_lens"):
        assert torch.equal(plain[k], fed[k]), k


# ---- host validation ------------------------------------------------------------------------------------------------

def test_token_table_layout_and_constant_rows(conf):
    T = 4
    t = prosody_table(2, duration_scale=[[1.0, 2.0, 0.5, 1.0], [1.0] * 4], pitch_shift=3.0, config=conf, T=T)
    assert t.shape == (2, T, 5) and t.dtype == torch.float32 and t.is_contiguous()
    per_item = prosody_table(2, duration_scale=[1.0, 1.0], pitch_shift=3.0, config=conf)
    assert torch.equal(t[1], per_item[1].expand(T, 5))
    assert t[0, :, 0].tolist() == [1.0, 2.0, 0.5, 1.0]
    # constant rows are exactly the per-item rows; an all-neutral table is no table at all
    kw = dict(duration_scale=[0.8, 1.25], pitch_shift=[4.0, -2.0], energy_scale=[1.3, 0.7])
    rows = {k: np.repeat(np.asarray(v)[:, None], T, axis=1) for k, v in kw.items()}
    assert torch.equal(prosody_table(2, config=conf, T=T, **rows), prosody_table(2, config=conf, **kw).unsqueeze(1).expand(2, T, 5))
    assert prosody_table(2, torch.ones(2, T), np.zeros((2, T)), [[1.0] * T] * 2, config=conf, T=T) is None


@pytest.mark.parametrize("kw", [
    dict(duration_scale=[[1.0, 0.0, 1.0], [1.0] * 3]), dict(duration_scale=[[1.0, math.nan, 1.0], [1.0] * 3]),
    dict(duration_scale=[[1.0, 20.0, 1.0], [1.0] * 3]), dict(duration_scale=[[1.0, 0.05, 1.0], [1.0] * 3]),
    dict(energy_scale=[[1.0, -1.0, 1.0], [1.0] * 3]), dict(pitch_shift=[[0.0, math.inf, 0.0], [0.0] * 3]),
    dict(pitch_shift=np.zeros((2, 4))), dict(duration_scale=np.ones((3, 3))), dict(energy_scale=np.ones((2, 3, 1))),
    dict(duration_scale=torch.ones(2, 3, device="meta")),
], ids=lambda kw: "%s%s" % (next(iter(kw)), np.shape(next(iter(kw.values())))))
def test_token_table_rejects_bad_values(kw):
    with pytest.raises(ValueError):
        prosody_table(2, T=3, **kw)


def test_constant_rows_keep_the_per_item_range():
    """Only rows that vary are held to [1/16, 16]: a row with one value throughout is a per-item scale."""
    t = prosody_table(2, duration_scale=[[0.01] * 3, [1.0, 2.0, 4.0]], T=3)
    assert t[0, :, 0].tolist() == [np.float32(0.01)] * 3
    with pytest.raises(ValueError, match="1/16"):
        prosody_table(2, duration_scale=[[0.01, 0.01, 1.0], [1.0] * 3], T=3)


def test_caller_values_shapes_and_dtypes():
    d = caller_values("durations", [[1, 2, 3]], 1, 3, "cpu", True)
    assert d.dtype == torch.int64 and d.shape == (1, 3)
    assert torch.equal(caller_values("durations", np.array([1, 2, 3], dtype=np.int32), 1, 3, "cpu", True), d)   # (T,) at B = 1
    p = caller_values("pitch", torch.tensor([0.5, 1.0, -1.0], dtype=torch.float64), 1, 3, "cpu", False)
    assert p.dtype == torch.float32 and p.shape == (1, 3)
    assert caller_values("energy", None, 2, 3, "cpu", False) is None
    bad = [("durations", [[1, -2, 3]], 1, True), ("durations", [[1.0, 2.0, 3.0]], 1, True), ("durations", [[1, 2]], 1, True),
           ("durations", [1, 2, 3, 4, 5, 6], 2, True), ("pitch", [[1, 2, 3]], 1, False), ("pitch", [[0.0, math.nan, 0.0]], 1, False),
           ("energy", [[0.0, math.inf, 0.0]], 1, False), ("energy", np.zeros((1, 3, 1), np.float32), 1, False),
           ("durations", torch.ones(1, 3, dtype=torch.int64, device="meta"), 1, True)]
    for name, v, B, integer in bad:
        with pytest.raises(ValueError):
            caller_values(name, v, B, 3, "cpu", integer)


def test_forward_validates_before_touching_the_engine(conf):
    """A bad (B,T) control or caller value raises ValueError where there is no GPU: nothing is packed or enqueued first."""
    m = JETSGenerator(conf)
    batch = synth.make_batch([5, 7])
    T = int(batch["inputs_ling"].shape[1])
    for kw in (dict(duration_scale=np.ones((2, T + 1))), dict(pitch_shift=np.full((2, T), math.nan)),
               dict(duration_scale=np.full((2, T), 0.5) + np.eye(2, T) * 30), dict(durations=-np.ones((2, T), np.int64)),
               dict(durations=np.ones((2, T), np.float32)), dict(pitch=np.ones(T, np.float32)), dict(energy=[[1.0] * T]),
               dict(durations=np.ones((2, T), np.int64), pitch=np.ones((2, T), np.int64))):
        with pytest.raises(ValueError):
            m(**batch, **kw)
        with pytest.raises(ValueError):
            m.am(**batch, **kw)
    assert m._ev_engine is None
    with pytest.raises(RuntimeError, match="no CPU fallback"):        # valid controls reach the engine as usual
        m(**batch, duration_scale=np.full((2, T), 0.9), durations=np.ones((2, T), np.int64), pitch=np.zeros((2, T)))
    with pytest.raises(NotImplementedError):
        m(**batch, mel_targets=torch.zeros(2, 10, 80), durations=np.ones((2, T), np.int64))


def test_new_symbols_are_declared_and_exported(lib):
    for name in ("ev_am_phase1_controls", "ev_op_duration_scan_controls"):
        assert name in _abi.SIGNATURES
        assert getattr(lib, name) is not None


def test_header_documents_the_new_status_bit():
    import os
    with open(os.path.join(os.path.dirname(_abi.__file__), "..", "include", "emotivoice_b200.h")) as f:
        h = f.read()
    assert "EV_API int ev_am_phase1_controls(" in h and "(B,T,5)" in h and "value 16" in h


# ---- front door -----------------------------------------------------------------------------------------------------

def test_phoneme_controls_validate_and_map_speed():
    assert fd.phoneme_controls(3) == fd.NEUTRAL_CONTROLS
    ds, ps, es = fd.phoneme_controls(3, speed=[1.0, 2.0, 0.5], pitch_shift=1.0)
    assert ds.tolist() == [1.0, 0.5, 2.0] and ps == 1.0 and es == 1.0
    for kw in (dict(speed=[1.0, 2.0]), dict(speed=[1.0, 0.0, 1.0]), dict(speed=[1.0, 20.0, 1.0]), dict(pitch_shift=[0.0, math.nan, 0.0]),
               dict(energy_scale=[1.0, 1.0, -1.0]), dict(speed=np.ones((3, 1)))):
        with pytest.raises(ValueError):
            fd.phoneme_controls(3, **kw)
    assert fd.given_values(2, durations=[1, 0], pitch=[0.5, 1.5])["durations"].dtype == np.int64
    for kw in (dict(durations=[1, -1]), dict(durations=[1.5, 1.0]), dict(pitch=[1.0]), dict(energy=[math.nan, 0.0])):
        with pytest.raises(ValueError):
            fd.given_values(2, **kw)


def test_collate_pads_per_phoneme_controls_and_caller_values():
    z = np.zeros(8, np.float32)
    items = [(np.array([1, 2]), 0, z, z, fd.phoneme_controls(2, speed=[1.0, 2.0])),
             (np.array([3, 4, 5]), 1, z, z, fd.speech_controls(speed=0.5, pitch_shift=-3.0)),
             (np.array([6]), 2, z, z)]
    b = fd.collate(items)
    assert b["duration_scale"].tolist() == [[1.0, 0.5, 1.0], [2.0, 2.0, 2.0], [1.0, 1.0, 1.0]]
    assert b["pitch_shift"].tolist() == [[0.0, 0.0, 0.0], [-3.0] * 3, [0.0] * 3]
    assert b["energy_scale"].tolist() == [[1.0] * 3] * 3
    given = [(np.array([1, 2]), 0, z, z, fd.NEUTRAL_CONTROLS, fd.given_values(2, durations=[3, 0], pitch=[0.5, -0.5])),
             (np.array([3, 4, 5]), 1, z, z, fd.NEUTRAL_CONTROLS, fd.given_values(3, durations=[1, 2, 3], pitch=[1.0, 2.0, 3.0]))]
    b = fd.collate(given)
    assert "duration_scale" not in b
    assert b["durations"].dtype == torch.int64 and b["durations"].tolist() == [[3, 0, 0], [1, 2, 3]]
    assert b["pitch"].dtype == torch.float32 and b["pitch"].tolist() == [[0.5, -0.5, 0.0], [1.0, 2.0, 3.0]]
    with pytest.raises(ValueError, match="same caller tracks"):
        fd.collate(given + [(np.array([7]), 0, z, z)])


def _fake_model(calls):
    def forward(inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding, **kw):
        calls.append(sorted(kw))
        B = inputs_ling.shape[0]
        n = [int(v) for v in input_lengths]
        d = kw.get("durations")
        frames = [int(d[b, :n[b]].sum()) if d is not None else 2 * n[b] for b in range(B)]
        wav = torch.zeros(B, 1, max(frames) * 256)
        for b in range(B):
            wav[b, 0, :frames[b] * 256] = float(inputs_speaker[b])
        return {"wav_predictions": wav, "mel_lengths": torch.tensor(frames, dtype=torch.int32)}
    return forward


def test_microbatcher_groups_requests_by_caller_tracks():
    calls = []
    z = np.zeros(8, np.float32)
    reqs = [dict(speed=[1.0, 2.0, 1.0]), dict(durations=[1, 2, 3]), dict(), dict(durations=[4, 0, 1], pitch_shift=[0.0, 2.0, 0.0])]
    with fd.MicroBatcher(_fake_model(calls), max_batch=4, max_wait_s=0.5) as mb:
        barrier = threading.Barrier(len(reqs))
        futs = [None] * len(reqs)

        def worker(i):
            barrier.wait()
            futs[i] = mb.submit(np.arange(1, 4), i, z, z, **reqs[i])

        ths = [threading.Thread(target=worker, args=(i,)) for i in range(len(reqs))]
        [t.start() for t in ths]
        [t.join() for t in ths]
        outs = [f.result(timeout=10) for f in futs]
        with pytest.raises(ValueError):
            mb.submit(np.arange(3), 0, z, z, durations=[1, -1, 1])
        with pytest.raises(ValueError):
            mb.submit(np.arange(3), 0, z, z, speed=[1.0, 1.0])
    assert mb.batches_run == 2 and len(calls) == 2
    assert sorted(calls) == sorted([["duration_scale", "energy_scale", "pitch_shift"],
                                    ["duration_scale", "durations", "energy_scale", "pitch_shift"]])
    for i, w in enumerate(outs):
        frames = 6 if "durations" not in reqs[i] else sum(reqs[i]["durations"])
        assert w.shape == (frames * 256,) and torch.all(w == i)
