"""Inputs and ABI-built chains shared by the GPU tests of the output stages (test_loudness_gpu, test_limiter_gpu, test_flac_gpu):
padded batches of signals, the engine's outputs of the fixture utterances, and ev_loudness / ev_limit called straight through
the ABI, which ``format_audio`` is checked against bit for bit."""
import numpy as np
import torch

from conftest import load_golden
from emotivoice_b200 import _abi, audio
from emotivoice_b200 import frontdoor as fd

SR = 16000
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
_cache = {}


def ten_minutes():
    """A 10-minute item: noise whose level moves slowly over 8 dB."""
    n = 600 * SR
    t = np.arange(n) / SR
    env = 10.0 ** ((-30.0 + 4.0 * np.sin(2 * np.pi * t / 47.0)) / 20.0)
    return np.clip(env * np.random.default_rng(8).standard_normal(n), -1.0, 1.0).astype(np.float32)


def padded_batch(signals, poison=True):
    """(B, 1, L) float32 host array, NaN past each item's length, and the lengths."""
    lens = [len(s) for s in signals]
    w = np.full((len(signals), 1, max(lens) + 37), np.nan if poison else 0.0, dtype=np.float32)
    for b, s in enumerate(signals):
        w[b, 0, :len(s)] = s
    return w, lens


def out_dict(w, lens, dev):
    """A forward's output dict holding the waveforms ``w`` with ``lens`` valid samples each (format them with hop=1)."""
    return {"wav_predictions": torch.from_numpy(w).to(dev), "mel_lengths_host": torch.tensor(lens, dtype=torch.int32)}


def engine_outputs(model, dev):
    """name -> (out, waveforms as host arrays) for b1_t100, b3_padded and the joined paragraph."""
    if not _cache:
        for name in ("b1_t100", "b3_padded"):
            g = load_golden(name)
            out = model(**{k: g[k].to(dev) for k in KEYS})
            wav = out["wav_predictions"].cpu().numpy()
            _cache[name] = (out, [wav[b, 0, :int(n) * 256] for b, n in enumerate(out["mel_lengths_host"].tolist())])
        g = load_golden("joined_paragraph")
        ends = np.cumsum(g["seg_lens"].numpy())
        segs = [g["ids"].numpy()[e - n:e] for e, n in zip(ends, g["seg_lens"].tolist())]
        batch = fd.collate([(s, int(spk), st.numpy(), ct.numpy()) for s, spk, st, ct in zip(segs, g["speakers"], g["style"], g["content"])])
        out = model(**{k: batch[k].to(dev) for k in KEYS}, join=[0] * len(segs))
        wav = out["wav_predictions"].cpu().numpy()
        _cache["paragraph"] = (out, [wav[0, 0, :int(out["joined_lengths_host"][0]) * 256]])
    return _cache


def abi_loudness(lib, dev, w, lens, items=None, target=-23.0):
    """ev_loudness straight through the ABI -> host (lufs, peak, gain) float32 arrays."""
    wt = torch.from_numpy(w).to(dev)
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    k = len(lens) if items is None else len(items)
    it = None if items is None else torch.tensor(items, dtype=torch.int64, device=dev)
    res = torch.empty((3, k), dtype=torch.float32, device=dev)
    kc = audio.k_weighting(SR)
    nb = lib.ev_loudness_workspace_bytes(k, wt.stride(0), SR)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_loudness(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None if it is None else it.data_ptr(), k, SR,
                               kc.ctypes.data, target, res[0].data_ptr(), res[1].data_ptr(), res[2].data_ptr(), ws.data_ptr(), nb,
                               torch.cuda.current_stream(dev).cuda_stream))
    r = res.cpu().numpy()
    return r[0], r[1], r[2]


def abi_limit(lib, dev, w, lens, rate, ceiling, lufs0=None, lufs1=None, target=-23.0, items=None):
    """ev_limit straight through the ABI -> host (k, stride) float32."""
    wt = torch.from_numpy(w).to(dev) if isinstance(w, np.ndarray) else w
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    k = len(lens) if items is None else len(items)
    it = None if items is None else torch.tensor(items, dtype=torch.int64, device=dev)
    bank, hold = audio.limit_bank(SR, rate)
    bank = torch.from_numpy(bank).to(dev)
    L = audio.limit_lookahead(SR)
    out = torch.full((k, wt.stride(0)), np.nan, dtype=torch.float32, device=dev)
    nb = lib.ev_limit_workspace_bytes(k, wt.stride(0), L)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    l0 = None if lufs0 is None else torch.from_numpy(np.asarray(lufs0, np.float32)).to(dev)
    l1 = None if lufs1 is None else torch.from_numpy(np.asarray(lufs1, np.float32)).to(dev)
    _abi.check(lib.ev_limit(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None if it is None else it.data_ptr(), k, SR,
                            None if l0 is None else l0.data_ptr(), None if l1 is None else l1.data_ptr(), target, ceiling,
                            bank.data_ptr(), bank.shape[0], bank.shape[1], L, hold, audio.limit_release(SR), out.data_ptr(),
                            out.stride(0), ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    return out.cpu().numpy()
