"""Long text on the GPU (``JETSGenerator.forward(join=...)``): the joined path against the fixtures of the unmodified reference
(oracle/make_golden_joined.py), the bitwise identities that need no oracle in all four precision modes (the joined pass is the
engine's own vocoder on the joined mel; one group per item is the plain forward; groups are batch-invariant), errors raised
before anything is enqueued or at the one sync, and PCM16 output."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import _abi, synth
from emotivoice_b200 import frontdoor as fd

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
PRED_KEYS = ("dec_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions", "mel_lengths")
MEL_TOL, WAV_TOL = 1e-4, 1e-4          # as test_e2e_gpu.py
MODES = ["fp32", "tf32", "bf16", "fp32_ffma"]


def _items(name):
    g = load_golden("joined_" + name)
    ends = np.cumsum(g["seg_lens"].numpy())
    segs = [g["ids"].numpy()[e - n:e] for e, n in zip(ends, g["seg_lens"].tolist())]
    return g, [(s, int(spk), st.numpy(), ct.numpy()) for s, spk, st, ct in zip(segs, g["speakers"], g["style"], g["content"])]


def _short(seed, n):
    b = synth.make_batch([n], seed=seed)
    return (b["inputs_ling"][0].numpy(), int(b["inputs_speaker"][0]), b["inputs_style_embedding"][0].numpy(),
            b["inputs_content_embedding"][0].numpy())


def _run(model, dev, items, **kw):
    batch = fd.collate(items)
    out = model(**{k: batch[k].to(dev) for k in KEYS}, **kw)
    torch.cuda.synchronize()
    return out


class _Precision:
    def __init__(self, model, mode):
        self.model, self.mode = model, mode

    def __enter__(self):
        self.model.precision = self.mode

    def __exit__(self, *exc):
        self.model.precision = "fp32"


@pytest.mark.parametrize("name", ["paragraph", "styles"])
def test_joined_forward_matches_reference_fixture(model, dev, name):
    g, items = _items(name)
    S = len(items)
    out = _run(model, dev, items, join=[0] * S)
    lens = g["mel_lens"].tolist()
    assert out["mel_lengths"].cpu().tolist() == lens
    off = np.concatenate([[0], np.cumsum(lens)])
    d_off = np.concatenate([[0], np.cumsum(g["seg_lens"].numpy())])
    for b in range(S):
        n = int(g["seg_lens"][b])
        assert torch.equal(out["log_duration_predictions"][b, :n].cpu(), g["durations"][d_off[b]:d_off[b + 1]])
        assert rel_max(out["dec_outputs"][b, :lens[b]].cpu(), g["joined_mel"][off[b]:off[b + 1]]) <= MEL_TOL
    total = int(off[-1])
    assert out["joined_lengths_host"].tolist() == [total] and out["joined_lengths"].cpu().tolist() == [total]
    assert tuple(out["joined_mel"].shape) == (1, total, 80) and tuple(out["wav_predictions"].shape) == (1, 1, 256 * total)
    n = g["wav_windows"].shape[1]                             # the fixture keeps the waveform at both ends and around each seam
    wav = torch.stack([out["wav_predictions"][0, 0, s:s + n].cpu() for s in g["wav_starts"].tolist()])
    e_mel, e_wav = rel_max(out["joined_mel"][0].cpu(), g["joined_mel"]), rel_rms(wav, g["wav_windows"])
    print(name, "joined mel rel-max %.2e wav rms-rel %.2e" % (e_mel, e_wav))
    assert e_mel <= MEL_TOL and e_wav <= WAV_TOL


@pytest.mark.parametrize("mode", MODES)
def test_joined_forward_is_the_engines_own_vocoder_and_the_plain_forward(model, dev, mode):
    _, para = _items("paragraph")
    _, styles = _items("styles")
    items = [_short(5, 17)] + para + styles[:2]
    B = len(items)
    join = [0, 1, 1, 1, 1, 1, 2, 2]
    with _Precision(model, mode):
        out = _run(model, dev, items, join=join)
        plain = _run(model, dev, items)
        for k in PRED_KEYS:                                  # the acoustic model runs exactly as without join
            assert torch.equal(out[k], plain[k]), k
        jl = out["joined_lengths_host"]
        glen = [sum(int(plain["mel_lengths"][b]) for b in range(B) if join[b] == g) for g in range(3)]
        assert jl.tolist() == glen and out["joined_lengths"].cpu().tolist() == glen
        mel = out["joined_mel"]
        assert tuple(mel.shape) == (3, max(glen), 80)
        m = plain["dec_outputs"]
        rows = [torch.cat([m[b, :int(plain["mel_lengths"][b])] for b in range(B) if join[b] == g]) for g in range(3)]
        for g in range(3):                                   # the gather: valid rows in item order, zeros after
            assert torch.equal(mel[g, :glen[g]], rows[g]) and torch.count_nonzero(mel[g, glen[g]:]) == 0
        eng = model._engine()
        with eng.call_lock:
            direct = eng.vocode(mel, time_major=True, mel_lens_ptr=out["joined_lengths"].data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(out["wav_predictions"], direct)
        one_each = _run(model, dev, items, join=range(B))
        for k in PRED_KEYS + ("wav_predictions",):
            assert torch.equal(one_each[k], plain[k]), k
        assert torch.equal(one_each["joined_lengths_host"], plain["mel_lengths_host"])


def test_groups_are_batch_invariant(model, dev):
    _, para = _items("paragraph")
    _, styles = _items("styles")
    groups = [[_short(7, 12)], para, styles, [_short(8, 31)]]
    items = [it for grp in groups for it in grp]
    join = [g for g, grp in enumerate(groups) for _ in grp]
    out = _run(model, dev, items, join=join)
    for g, grp in enumerate(groups):
        alone = _run(model, dev, grp, join=[0] * len(grp))
        n = int(alone["joined_lengths_host"][0])
        assert int(out["joined_lengths_host"][g]) == n
        assert torch.equal(out["joined_mel"][g, :n], alone["joined_mel"][0])
        assert torch.equal(out["wav_predictions"][g, 0, :256 * n], alone["wav_predictions"][0, 0])
        assert torch.count_nonzero(out["wav_predictions"][g, 0, 256 * n:]) == 0


def test_errors_raise_and_the_model_keeps_serving(model, dev):
    items = [_short(9, 20), _short(10, 25), _short(11, 14)]
    n0 = _abi.launch_count()
    for bad in ([0, 2, 2], [1, 1, 1], [0, 1], [0.0, 0.0, 1.0]):
        with pytest.raises(ValueError):
            _run(model, dev, items, join=bad)
    model.compat_padded_batch = True
    try:
        with pytest.raises(ValueError):
            _run(model, dev, items, join=[0, 0, 0])
    finally:
        model.compat_padded_batch = False
    assert _abi.launch_count() == n0                            # nothing enqueued
    with pytest.raises(RuntimeError):                           # a segment scaled to zero frames
        _run(model, dev, items, join=[0, 0, 1], duration_scale=[1.0, 1e-4, 1.0])
    T = 25                                                      # a joined output too long for the vocoder's int32 sample index
    dur = torch.zeros(3, T, dtype=torch.int64)
    dur[0, :20], dur[1, :25] = 250_000, 250_000                 # 5M + 6.25M frames: each item fits, their group does not
    dur[2, :14] = 3
    with pytest.raises(ValueError, match="joined output"):
        _run(model, dev, items, join=[0, 0, 1], durations=dur)
    out = _run(model, dev, items, join=[0, 0, 1])
    plain = _run(model, dev, items)
    assert torch.equal(out["dec_outputs"], plain["dec_outputs"])


def test_fetch_pcm16_trims_joined_outputs(model, dev):
    _, para = _items("paragraph")
    items = [_short(12, 15)] + para
    out = _run(model, dev, items, join=[0] + [1] * len(para))
    pcm = fd.fetch_pcm16(model, out)
    full = model.to_pcm16(out["wav_predictions"]).cpu()
    assert len(pcm) == 2
    for g in range(2):
        n = int(out["joined_lengths"][g]) * 256
        assert np.array_equal(pcm[g], full[g, 0, :n].numpy())
