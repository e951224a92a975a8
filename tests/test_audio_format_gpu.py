"""Output formats on the GPU (``JETSGenerator.format_audio`` / ``frontdoor.fetch_audio``, ev_format_audio): resampling against
scipy's resample_poly in float64, PCM16 and G.711 against their definitions, the source rate bit for bit, batch independence,
item edges, poisoned padding, joined outputs, mixed formats in one MicroBatcher forward, and argument errors."""
import numpy as np
import pytest
import torch
from scipy.signal import firwin, resample_poly

from audio_cases import out_dict
from conftest import GOLDEN, load_golden
from emotivoice_b200 import _abi, audio, synth
from emotivoice_b200 import frontdoor as fd

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 96000, 192000]
TAU = 2.0 ** -16
_cache = {}


def _g711():
    z = np.load(GOLDEN + "/g711.npz")
    return {"mulaw": z["ulaw"], "alaw": z["alaw"]}


def _engine_out(model, dev, name="b3_padded"):
    """A fixture batch through the engine: b3_padded (three items of mixed lengths) or b1_t100 (one utterance of 537 frames)."""
    if name not in _cache:
        g = load_golden(name)
        _cache[name] = (g, model(**{k: g[k].to(dev) for k in KEYS}))
    return _cache[name]


def _items(out):
    wav = out["wav_predictions"].cpu().numpy()
    return [wav[b, 0, :int(n) * 256] for b, n in enumerate(out["mel_lengths_host"].tolist())]


def _reference(x, up, down):
    """resample_poly of x in float64 and m = the sum of |tap * sample| entering each output."""
    x64 = np.asarray(x, dtype=np.float64)
    y64 = resample_poly(x64, up, down)
    if up == down == 1:
        return y64, np.abs(x64)
    mx = max(up, down)
    m = resample_poly(np.abs(x64), up, down, window=np.abs(firwin(20 * mx + 1, 1.0 / mx, window=("kaiser", 5.0))))
    return y64, m


def _pcm16_ref(y64):
    return np.trunc(np.clip(y64 * 32768.0, -32768.0, 32767.0)).astype(np.int64)


def _check_float32(got, y64, m):
    assert got.dtype == np.float32 and got.shape == y64.shape
    err = np.abs(got.astype(np.float64) - y64)
    assert np.all(err <= TAU * m + 1e-30), (err.max(), (err / np.maximum(m, 1e-30)).max())


def _check_pcm16(got, y64, m):
    assert got.dtype == np.int16 and got.shape == y64.shape
    want = _pcm16_ref(y64)
    d = np.abs(got.astype(np.int64) - want)
    assert d.max(initial=0) <= 1
    s = y64 * 32768.0
    near = np.abs(s - np.round(s)) <= TAU * m * 32768.0
    assert np.array_equal(got[~near], want[~near])


@pytest.mark.parametrize("name", ["b3_padded", "b1_t100"])
@pytest.mark.parametrize("rate", RATES)
def test_engine_waveform_matches_resample_poly_in_float64(model, dev, rate, name):
    _, out = _engine_out(model, dev, name)
    _, up, down = audio.plan(rate, "pcm16", 16000)
    xs = _items(out)
    f32 = fd.fetch_audio(model, out, rate, "float32")
    pcm = fd.fetch_audio(model, out, rate, "pcm16")
    tables = _g711()
    for b, x in enumerate(xs):
        y64, m = _reference(x, up, down)
        _check_float32(f32[b], y64, m)
        _check_pcm16(pcm[b], y64, m)
        for enc in ("mulaw", "alaw"):
            codes = fd.fetch_audio(model, out, rate, enc, items=[b])[0]
            assert codes.dtype == np.uint8 and np.array_equal(codes, tables[enc][pcm[b].astype(np.int64) + 32768])


def test_source_rate_is_bitwise_the_trimmed_waveform_and_to_pcm16(model, dev):
    _, out = _engine_out(model, dev)
    xs = _items(out)
    full = model.to_pcm16(out["wav_predictions"]).cpu().numpy()
    f32 = fd.fetch_audio(model, out, None, "float32")
    pcm = fd.fetch_audio(model, out)
    legacy = fd.fetch_pcm16(model, out)
    for b, x in enumerate(xs):
        assert np.array_equal(f32[b].view(np.int32), x.view(np.int32))
        assert np.array_equal(pcm[b], full[b, 0, :len(x)]) and np.array_equal(legacy[b], pcm[b])
        assert np.array_equal(pcm[b], (x * 32768.0).astype("int16"))
    packed, offs = model.format_audio(out, 16000, "pcm16")
    assert packed.dtype == torch.int16 and packed.device == dev and offs.tolist() == np.cumsum([0] + [len(x) for x in xs]).tolist()


def test_engine_batch_gives_each_item_its_b1_output(model, dev):
    g, out = _engine_out(model, dev)
    for b in range(3):
        single = model(**{k: v.to(dev) for k, v in synth.slice_batch(g, b).items()})
        for rate, enc in ((8000, "mulaw"), (44100, "float32"), (24000, "pcm16")):
            assert np.array_equal(fd.fetch_audio(model, single, rate, enc)[0], fd.fetch_audio(model, out, rate, enc, items=[b])[0])


def _synthetic(lens, seed=0, poison=True):
    """(B,1,L) waveform, values in (-1, 1) up to each length and NaN after it; the lengths go in as mel_lengths_host with hop 1."""
    rng = np.random.default_rng(seed)
    L = max(lens) + 37
    w = np.full((len(lens), 1, L), np.nan if poison else 0.0, dtype=np.float32)
    for b, n in enumerate(lens):
        w[b, 0, :n] = np.tanh(rng.standard_normal(n) * 0.8).astype(np.float32)
    return w


@pytest.mark.parametrize("rate", [8000, 11025, 24000, 44100, 48000, 192000])
def test_item_edges_poisoned_padding_and_batch_independence(model, dev, rate):
    _, up, down = audio.plan(rate, "float32", 16000)
    lens = [1, 2, 3000]
    for t in (256, 512):                  # outputs that end just before, on and just after a tile edge (256 outputs per tile)
        lens += [(t * down) // up + d for d in (-1, 0, 1, 2)]
    w = _synthetic(lens, seed=rate)
    out = out_dict(w, lens, dev)
    for enc in ("float32", "pcm16", "mulaw"):
        allv = fd.fetch_audio(model, out, rate, enc, hop=1)
        assert [len(a) for a in allv] == [audio.resampled_length(n, up, down) for n in lens]
        for b, n in enumerate(lens):
            alone = fd.fetch_audio(model, out_dict(np.ascontiguousarray(w[b:b + 1, :, :n + 5]), [n], dev), rate, enc, hop=1)[0]
            assert np.array_equal(alone, allv[b]), (enc, b, n)
            if enc == "float32":
                assert not np.isnan(allv[b]).any()
                y64, m = _reference(w[b, 0, :n], up, down)
                _check_float32(allv[b], y64, m)
            elif enc == "pcm16":
                y64, m = _reference(w[b, 0, :n], up, down)
                _check_pcm16(allv[b], y64, m)
    f32 = fd.fetch_audio(model, out, rate, "float32", hop=1)
    rev = fd.fetch_audio(model, out, rate, "float32", items=list(range(len(lens)))[::-1], hop=1)
    assert all(np.array_equal(a, f) for a, f in zip(rev[::-1], f32))


def test_joined_forward_formats_one_output_per_group(model, dev):
    items = []
    for seed, n in ((21, 17), (22, 30), (23, 12)):
        bt = synth.make_batch([n], seed=seed)
        items.append((bt["inputs_ling"][0].numpy(), int(bt["inputs_speaker"][0]), bt["inputs_style_embedding"][0].numpy(),
                      bt["inputs_content_embedding"][0].numpy()))
    batch = fd.collate(items)
    out = model(**{k: batch[k].to(dev) for k in KEYS}, join=[0, 0, 1])
    wav = out["wav_predictions"].cpu().numpy()
    glen = out["joined_lengths_host"].tolist()
    got = fd.fetch_audio(model, out, 24000, "float32")
    pcm = fd.fetch_audio(model, out)
    assert len(got) == len(pcm) == 2
    for g in range(2):
        x = wav[g, 0, :glen[g] * 256]
        y64, m = _reference(x, 3, 2)
        _check_float32(got[g], y64, m)
        assert np.array_equal(pcm[g], (x * 32768.0).astype("int16"))


def test_microbatcher_mixed_formats_equal_fetch_audio_alone(model, dev):
    rng = np.random.default_rng(31)
    utts = [synth.make_utterance(rng, int(n)) for n in (14, 33, 9, 21, 17)]
    fmts = [(24000, "pcm16"), (8000, "mulaw"), (44100, "float32"), (None, "alaw"), (None, None)]
    with fd.MicroBatcher(model, device=dev, max_batch=5, max_wait_s=0.5) as mb:
        futs = [mb.submit(u["ids"], int(u["speaker"]), u["style"], u["content"], sample_rate=r, encoding=e)
                for u, (r, e) in zip(utts, fmts)]
        got = [f.result(timeout=120) for f in futs]
        assert mb.batches_run <= 2
    for u, (r, e), w in zip(utts, fmts, got):
        single = model(**fd.collate([(u["ids"], int(u["speaker"]), u["style"], u["content"])], dev))
        if e is None:
            assert torch.equal(single["wav_predictions"][0, 0].cpu(), w)
        else:
            want = fd.fetch_audio(model, single, r, e)[0]
            assert w.dtype == want.dtype and np.array_equal(w, want), (r, e)


def test_launches_per_chain_shape(model, dev):
    """format_audio enqueues its stages and nothing else: ev_format_audio 1, ev_loudness 2, ev_limit 3 per pass, ev_flac_encode
    4; no launch when every listed output is empty."""
    _, out = _engine_out(model, dev)
    empty = out_dict(np.zeros((2, 1, 64), np.float32), [0, 0], dev)
    for (loudness, true_peak), n in {(None, None): 1, (-16.0, None): 3, (None, -1.0): 4, (-16.0, -1.0): 11}.items():
        for enc, extra in (("pcm16", 0), ("flac", 4)):
            n0 = _abi.launch_count()
            model.format_audio(out, 24000, enc, loudness=loudness, true_peak=true_peak)
            assert _abi.launch_count() - n0 == n + extra, (loudness, true_peak, enc)
        n0 = _abi.launch_count()
        packed, offs = model.format_audio(empty, 24000, "pcm16", hop=1, loudness=loudness, true_peak=true_peak)
        assert _abi.launch_count() == n0 and packed.numel() == 0 and offs.tolist() == [0, 0, 0], (loudness, true_peak)


def test_invalid_arguments_raise_before_anything_is_enqueued(model, dev, lib):
    _, out = _engine_out(model, dev)
    w = out["wav_predictions"]
    n_in = torch.full((3,), 256, dtype=torch.int64, device=dev)
    off = torch.zeros(3, dtype=torch.int64, device=dev)
    dst = torch.empty(4096, dtype=torch.float32, device=dev)
    bank = torch.from_numpy(audio.polyphase_bank(3, 2)).to(dev)
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    for kw in (dict(sample_rate=44100.5), dict(sample_rate=3000), dict(sample_rate=16001), dict(encoding="mp3"),
               dict(items=[3]), dict(items=[]), dict(items=[-1])):
        with pytest.raises(ValueError):
            model.format_audio(out, **kw)
    with pytest.raises(ValueError):
        model.format_audio({"wav_predictions": out["wav_predictions"].double()})
    bad = [(bank.data_ptr(), 3, 2, 20, 0),         # taps_per_phase of another filter
           (bank.data_ptr(), 6, 4, 21, 0),         # not coprime
           (None, 3, 2, 21, 0),                    # no bank for a ratio
           (bank.data_ptr(), 1, 1, 21, 0),         # a bank for the copy
           (bank.data_ptr(), 3, 2, 21, 4),         # unknown encoding
           (bank.data_ptr(), 2048, 1, 21, 0)]      # factor above 1024
    for bk, up, down, taps, enc in bad:
        with pytest.raises(_abi.EvError):
            _abi.check(lib.ev_format_audio(w.data_ptr(), w.stride(0), n_in.data_ptr(), None, 3, off.data_ptr(), bk, up, down, taps,
                                           enc, dst.data_ptr(), None, torch.cuda.current_stream(dev).cuda_stream))
    assert _abi.launch_count() == n0
    got = fd.fetch_audio(model, out, 48000, "pcm16")
    assert [len(a) for a in got] == [3 * int(n) * 256 for n in out["mel_lengths_host"].tolist()]
