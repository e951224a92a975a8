"""Long text without a GPU: the phoneme splitter on the reference's inference text, the joined-path oracle against the fixtures
that oracle/make_golden_joined.py generated from the unmodified reference, host validation of ``join``, the micro-batcher's
joined requests with a fake model, and the new C symbol."""
import os
import threading

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max
from emotivoice_b200 import frontdoor as fd
from emotivoice_b200 import _abi
from emotivoice_b200.modules import join_groups, group_frames
from oracle import joined_oracle

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frontdoor")
SOS = fd.SOS_EOS


def _lines():
    with open(os.path.join(FIXTURES, "inference_text"), encoding="utf-8") as f:
        return [fd.parse_line(l).phonemes for l in f if l.strip()]


def _runs(toks):
    """The input's inner tokens, cut at inner <sos/eos>, as the splitter must see them."""
    if toks and toks[0] == SOS:
        toks = toks[1:]
    if toks and toks[-1] == SOS:
        toks = toks[:-1]
    runs, cur = [], []
    for t in toks:
        if t == SOS:
            if cur:
                runs.append(cur)
            cur = []
        else:
            cur.append(t)
    return runs + ([cur] if cur else [])


def _check_split(toks, m):
    segs = fd.split_phonemes(toks, max_phonemes=m)
    width = m - 2
    for s in segs:
        assert 3 <= len(s) <= m and s[0] == s[-1] == SOS and SOS not in s[1:-1]
    inner = [s[1:-1] for s in segs]
    assert [t for s in inner for t in s] == [t for r in _runs(toks) for t in r]
    k = 0                                     # every cut inside a run is at the window's last punctuation break, else last word break
    for run in _runs(toks):
        i = 0
        while i < len(run):
            seg = inner[k]
            assert run[i:i + len(seg)] == seg
            if i + len(seg) < len(run):
                window, rest = run[i:i + width], run[i + len(seg):i + width]
                if any(t in fd.PUNCTUATION_BREAKS for t in window):
                    assert seg[-1] in fd.PUNCTUATION_BREAKS and not any(t in fd.PUNCTUATION_BREAKS for t in rest)
                elif any(t in fd.WORD_BREAKS for t in window):
                    assert seg[-1] in fd.WORD_BREAKS and not any(t in fd.WORD_BREAKS for t in rest)
                else:
                    assert len(seg) == width
            i += len(seg)
            k += 1
    assert k == len(segs)
    return segs


def test_break_classes_are_tokens_of_the_reference_table():
    t2i = fd.load_symbol_table(os.path.join(FIXTURES, "tokenlist"))
    for name in fd.PUNCTUATION_BREAKS | fd.WORD_BREAKS | {SOS}:
        assert name in t2i, name
    assert not fd.PUNCTUATION_BREAKS & fd.WORD_BREAKS


@pytest.mark.parametrize("m", [8, 16, 32, 64, 256])
def test_split_guarantees_on_the_inference_text(m):
    lines = _lines()
    for toks in lines:
        segs = _check_split(toks, m)
        if len(toks) <= m:
            assert segs == [toks]                 # a line that fits comes back whole
    if m == 256:
        assert max(len(t) for t in lines) == 223
    joined = [t for toks in lines for t in toks]  # a paragraph of frontend lines falls apart at their edges (and further)
    segs = _check_split(joined, m)
    assert len(segs) >= len(lines)
    paragraph = [SOS] + [t for toks in lines for t in toks[1:-1]] + [SOS]
    _check_split(paragraph, m)


def test_split_edges_and_errors():
    assert fd.split_phonemes(["a", "b"], 8) == [[SOS, "a", "b", SOS]]          # unwrapped input gets wrapped
    assert fd.split_phonemes([SOS, "a", SOS, SOS, "b", SOS], 8) == [[SOS, "a", SOS], [SOS, "b", SOS]]
    assert fd.split_phonemes([SOS, "a", "b", "c", "d", SOS], 3) == [[SOS, t, SOS] for t in "abcd"]
    assert fd.split_phonemes([SOS, "a", "sp1", "b", "sp3", "c", "sp1", "d", SOS], 6) == [
        [SOS, "a", "sp1", "b", "sp3", SOS], [SOS, "c", "sp1", "d", SOS]]
    for bad in ([], [SOS], [SOS, SOS], [SOS, SOS, SOS]):
        with pytest.raises(ValueError):
            fd.split_phonemes(bad)
    with pytest.raises(ValueError):
        fd.split_phonemes([SOS, "a", SOS], max_phonemes=2)


# ---- the oracle against the reference fixtures ------------------------------------------------------------------------

def _segments(g):
    ends = np.cumsum(g["seg_lens"].numpy())
    return [g["ids"][e - n:e] for e, n in zip(ends, g["seg_lens"].tolist())]


@pytest.mark.parametrize("name", ["paragraph", "styles"])
def test_oracle_reproduces_joined_fixture(name, sd, conf):
    g = load_golden("joined_" + name)
    segs = _segments(g)
    S = len(segs)
    assert g["style"].shape == (S, 768) and g["speakers"].shape == (S,)
    if name == "paragraph":
        assert S == 5 and 220 <= int(g["seg_lens"].sum()) <= 250
    o = joined_oracle.joined_forward(sd, conf, segs, g["speakers"].tolist(), list(g["style"]), list(g["content"]))
    assert torch.equal(torch.cat([p["log_duration_predictions"][0] for p in o["per_segment"]]), g["durations"])
    assert [int(p["mel_lens"][0]) for p in o["per_segment"]] == g["mel_lens"].tolist()
    assert o["joined_mel"][0].shape == g["joined_mel"].shape
    assert rel_max(o["joined_mel"][0], g["joined_mel"]) <= 2e-6
    n = g["wav_windows"].shape[1]
    assert g["wav_starts"].numel() == S + 1 and int(g["wav_starts"][-1]) + n == 256 * int(g["mel_lens"].sum())
    wav = torch.stack([o["joined_wav"][0, 0, s:s + n] for s in g["wav_starts"].tolist()])
    assert rel_max(wav, g["wav_windows"]) <= 2e-6


# ---- host validation of join -------------------------------------------------------------------------------------------

def test_join_groups_validates_before_anything_runs():
    assert join_groups(None, 3) is None
    assert join_groups([0, 0, 1], 3).tolist() == [0, 0, 1] and join_groups(range(3), 3).dtype == np.int32
    assert join_groups(torch.tensor([0, 1, 1, 2]), 4).tolist() == [0, 1, 1, 2]
    for bad, B in (([1, 1], 2), ([0, 2], 2), ([0, 1, 0], 3), ([0, 0], 3), ([0.0, 1.0], 2), ([[0, 1]], 2), ("01", 2),
                   ([True, False], 2), ([0, [1]], 2)):
        with pytest.raises(ValueError):
            join_groups(bad, B)
    with pytest.raises(ValueError):
        join_groups(list(range(4097)), 4097)
    assert group_frames(np.array([0, 0, 1, 2, 2], np.int32), [3, 4, 5, 6, 7]).tolist() == [7, 5, 13]


def test_join_raises_without_a_gpu_before_anything_runs(conf):
    """join errors come from the host checks, ahead of the engine (which would need a GPU)."""
    from emotivoice_b200.modules import JETSGenerator
    m = JETSGenerator(conf).eval()
    x = dict(inputs_ling=torch.ones(2, 5, dtype=torch.int64), input_lengths=torch.tensor([5, 5]), inputs_speaker=torch.tensor([0, 1]),
             inputs_style_embedding=torch.zeros(2, 768), inputs_content_embedding=torch.zeros(2, 768))
    with pytest.raises(ValueError):
        m(**x, join=[0, 2])
    m.compat_padded_batch = True
    with pytest.raises(ValueError, match="compat_padded_batch"):
        m(**x, join=[0, 0])


def test_join_mel_symbol(lib):
    assert "ev_join_mel" in _abi.SIGNATURES and hasattr(lib, "ev_join_mel")
    assert lib.ev_join_mel(None, None, None, 1, 1, 80, 1, 1, None, None, None) == -1
    assert b"null" in lib.ev_last_error()


# ---- the micro-batcher -------------------------------------------------------------------------------------------------

def _fake_model(calls):
    """2 frames per phoneme; an item's signal is speaker + 1e-3 * sum of its ids; with join, each group's wav is its items'
    signals in order."""
    def forward(inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding, **kw):
        calls.append(dict(B=int(inputs_ling.shape[0]), kw=kw, style=inputs_style_embedding.clone()))
        B = inputs_ling.shape[0]
        mel = (input_lengths * 2).to(torch.int32)
        sig = [float(inputs_speaker[b]) + inputs_ling[b, :int(input_lengths[b])].sum().item() * 1e-3 for b in range(B)]
        join = kw.get("join", list(range(B)))
        G = join[-1] + 1
        glen = [sum(int(mel[b]) for b in range(B) if join[b] == g) for g in range(G)]
        wav = torch.zeros(G, 1, max(glen) * 256)
        pos = [0] * G
        for b in range(B):
            g, n = join[b], int(mel[b]) * 256
            wav[g, 0, pos[g]:pos[g] + n] = sig[b]
            pos[g] += n
        out = {"wav_predictions": wav, "mel_lengths": mel}
        if "join" in kw:
            out.update(joined_lengths=torch.tensor(glen, dtype=torch.int32), joined_lengths_host=torch.tensor(glen, dtype=torch.int32))
        return out
    return forward


def _vec(v):
    return np.full(768, v, np.float32)


def test_microbatcher_mixes_plain_and_joined_requests_in_one_forward():
    calls = []
    with fd.MicroBatcher(_fake_model(calls), max_batch=5, max_wait_s=2.0) as mb:
        f0 = mb.submit(np.array([1, 2]), 3, _vec(0), _vec(0))
        f1 = mb.submit_joined([np.array([1, 5]), np.array([1, 6, 7]), np.array([2])], 4, [_vec(1), _vec(2), _vec(3)], _vec(0))
        f2 = mb.submit(np.array([9]), 5, _vec(0), _vec(0), speed=2.0)
        w0, w1, w2 = (f.result(timeout=10) for f in (f0, f1, f2))
    assert len(calls) == 1 and calls[0]["B"] == 5 and calls[0]["kw"]["join"] == [0, 1, 1, 1, 2]
    assert calls[0]["kw"]["duration_scale"] == [1.0, 1.0, 1.0, 1.0, 0.5]
    assert calls[0]["style"][:, 0].tolist() == [0, 1, 2, 3, 0]                     # one prompt per segment
    assert torch.equal(w0, torch.full((4 * 256,), 3 + 3e-3))
    want = torch.cat([torch.full((4 * 256,), 4 + 6e-3), torch.full((6 * 256,), 4 + 14e-3), torch.full((2 * 256,), 4 + 2e-3)])
    assert torch.equal(w1, want)
    assert torch.equal(w2, torch.full((2 * 256,), 5 + 9e-3))


def test_microbatcher_without_joined_requests_makes_the_plain_call():
    calls = []
    with fd.MicroBatcher(_fake_model(calls), max_batch=2, max_wait_s=2.0) as mb:
        fs = [mb.submit(np.array([1, 2, 3]), i, _vec(0), _vec(0)) for i in range(2)]
        [f.result(timeout=10) for f in fs]
    assert len(calls) == 1 and calls[0]["kw"] == {}


def test_joined_request_larger_than_max_batch_runs_alone_and_is_never_split():
    calls = []
    gate = threading.Event()
    model = _fake_model(calls)

    def forward(**kw):
        gate.wait(10)
        return model(**kw)

    with fd.MicroBatcher(forward, max_batch=3, max_wait_s=0.05) as mb:
        fa = mb.submit(np.array([1]), 0, _vec(0), _vec(0))                  # occupies the worker until the gate opens
        fb = mb.submit_joined([np.array([1, 2])] * 5, 1, _vec(0), _vec(0))  # 5 segments > max_batch
        fc = mb.submit_joined([np.array([3])] * 2, 2, _vec(0), _vec(0))
        fd_ = mb.submit(np.array([4]), 3, _vec(0), _vec(0))
        gate.set()
        res = [f.result(timeout=10) for f in (fa, fb, fc, fd_)]
    sizes = [c["B"] for c in calls]
    assert sizes[0] == 1 and 5 in sizes and sum(sizes) == 1 + 5 + 2 + 1
    big = calls[sizes.index(5)]
    assert big["kw"]["join"] == [0] * 5                                       # alone, whole
    assert all(c["B"] <= 3 for c in calls if c is not big)
    assert res[1].shape == (5 * 4 * 256,) and res[2].shape == (2 * 2 * 256,)


def test_submit_joined_checks_its_arguments():
    with fd.MicroBatcher(_fake_model([]), max_batch=2) as mb:
        for bad in ([], [np.array([], np.int64)], [np.array([[1, 2]])]):
            with pytest.raises(ValueError):
                mb.submit_joined(bad, 0, _vec(0), _vec(0))
        with pytest.raises(ValueError):
            mb.submit_joined([np.array([1])] * 2, 0, [_vec(0)] * 3, _vec(0))
        with pytest.raises(ValueError):
            mb.submit_joined([np.array([1])], 0, _vec(0), _vec(0), speed=0.0)
        with pytest.raises(TypeError):
            mb.submit_joined([np.array([1])], 0, _vec(0), _vec(0), durations=[1])

