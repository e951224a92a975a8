"""Host side of the APIs that take a batch of recordings (``feats``, ``loudness.meter``, ``watermark.detect``,
``evaluate.compare``) and of the output chain: the checks of the waveform batch and its lengths, the pinned upload of host
integers, the per-device cache of constant tables, and resampling through ``ev_format_audio``.
"""
import collections.abc

import numpy as np
import torch

from . import _abi, audio

_TABLES = {}                    # (key, device) -> what device_table made for that key on that device


def host_lengths(lengths, B, L, name="lengths"):
    """The valid samples of each of B rows of L samples -> a list of B ints in [0, L].  ``lengths``: None (every row is L), a
    sequence or 1-D numpy array of Python or numpy integers, or a 1-D CPU integer tensor.  Anything else (floats, bools,
    strings, CUDA or meta tensors, a wrong count, a value out of range) raises ValueError, before any device work."""
    if lengths is None:
        return [L] * B
    if isinstance(lengths, np.ndarray) or (torch.is_tensor(lengths) and lengths.device.type == "cpu"):
        lengths = lengths.tolist()
    if (isinstance(lengths, (str, bytes)) or not isinstance(lengths, collections.abc.Sequence)     # np.bool_ is no np.integer
            or not all(type(v) is int or (isinstance(v, (int, np.integer)) and not isinstance(v, bool)) for v in lengths)):
        raise ValueError("%s must be %d host integers in [0, %d] (a sequence or a CPU tensor)" % (name, B, L))
    if len(lengths) != B:
        raise ValueError("%d %s for %d items" % (len(lengths), name, B))
    lens = [int(v) for v in lengths]
    bad = [n for n in lens if not 0 <= n <= L]
    if bad:
        raise ValueError("%s: %d is negative or exceeds the %d samples of a row" % (name, bad[0], L))
    return lens


def recording_batch(wav, name="wav"):
    """Checks a batch of recordings, one per row: a CUDA (B, L) float32 tensor with 1 <= B <= 65535 and L >= 1, else
    ValueError.  Returns it with each row's samples contiguous and rows that do not overlap, copying only when they are not
    (rows may be further apart than L)."""
    if not (isinstance(wav, torch.Tensor) and wav.dim() == 2 and wav.dtype == torch.float32 and wav.is_cuda):
        raise ValueError("%s must be a CUDA (B, L) float32 tensor" % name)
    B, L = int(wav.shape[0]), int(wav.shape[1])
    if not 1 <= B <= 65535 or L < 1:
        raise ValueError("%s must hold 1 to 65535 recordings of at least one sample, got shape %s" % (name, tuple(wav.shape)))
    return wav if wav.stride(1) == 1 and wav.stride(0) >= L else wav.contiguous()


def upload(arrays, dev, dtype=np.int64):
    """Host integer arrays -> one device tensor of the numpy ``dtype``, copied through pinned memory without blocking, and the
    device address of each array in it.  The tensor must stay referenced until the last launch that reads it has been
    enqueued."""
    t = torch.from_numpy(np.concatenate([np.asarray(a, dtype) for a in arrays])).pin_memory().to(dev, non_blocking=True)
    ptrs, p, size = [], t.data_ptr(), t.element_size()
    for a in arrays:
        ptrs.append(p)
        p += size * len(a)
    return t, ptrs


def _to(a, dev):
    if not isinstance(a, np.ndarray):
        return a
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t if torch.device(dev).type == "cpu" else t.pin_memory().to(dev, non_blocking=True)


def device_table(key, make, dev):
    """The constant table of ``key`` on ``dev``.  ``make()`` returns a host array, a tuple of host arrays and plain values,
    or None.  The first call for a key and device copies each array to ``dev`` through pinned memory without blocking (on
    the CPU it stays a host tensor); every later call returns the same objects."""
    k = (key, str(dev))
    if k not in _TABLES:
        t = make()
        _TABLES[k] = tuple(_to(a, dev) for a in t) if isinstance(t, tuple) else _to(t, dev)
    return _TABLES[k]


def polyphase_bank(up, down, dev):
    """``audio.polyphase_bank(up, down)``, the filter bank of ev_format_audio, on ``dev``: made once per device."""
    return device_table(("polyphase", up, down), lambda: audio.polyphase_bank(up, down), dev)


def resample(wav, lens, rate, target):
    """CUDA (B, L) float32 recordings at ``rate`` (each row's samples contiguous), host lengths ``lens`` -> ((B, L') float32
    at ``target`` Hz, the lengths at ``target``), through ev_format_audio's float32 path: each row's valid samples resampled
    as ``scipy.signal.resample_poly`` does.  The rates must be ones ``audio.plan`` accepts; a row is not written past its own
    valid samples.  No sync."""
    _, up, down = audio.plan(target, "float32", rate)
    B, L = wav.shape
    dev = wav.device
    out = torch.empty((B, audio.resampled_length(L, up, down)), dtype=torch.float32, device=dev)
    meta, (p_n, p_out) = upload([lens, [b * out.stride(0) for b in range(B)]], dev)     # n_in, where each row starts in out
    bank = polyphase_bank(up, down, dev)
    _abi.check(_abi.load().ev_format_audio(wav.data_ptr(), int(wav.stride(0)), p_n, None, B, p_out, bank.data_ptr(), up, down,
                                           int(bank.shape[1]), audio.ENCODINGS["float32"], out.data_ptr(), None,
                                           torch.cuda.current_stream(dev).cuda_stream))
    return out, [audio.resampled_length(n, up, down) for n in lens]
