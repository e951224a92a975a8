"""The caller-side plumbing either side of the hot path (SURVEY.md s8f rank 3): the
``<speaker>|<prompt>|<phoneme>|<content>`` input contract and a micro-batching queue.

Every reference front-end (inference_am_vocoder_joint.py:76-131, demo_page.py:119-150,
openaiapi.py:110-142) does the same four things around ``generator(...)``: read the symbol tables,
split the 4-field line, map phonemes / speaker to ids, and run B=1.  This module restates that
plumbing for hosts that want it without the reference scripts, and adds what turns batch throughput
into served throughput: a queue that groups concurrent requests into one padded forward.  Because the
engine's batches are bitwise equal to B=1 runs (DESIGN.md s1), micro-batching is invisible to callers.

Pure host code: no CUDA, no torch ops beyond tensor construction.  The style / content vectors come
from the caller (the simbert encoder is out of scope, SURVEY.md s2 row 17).

Prompt side (s8f rank 1): ``PromptEmbeddingCache`` -- batched, cached ``get_style_embedding``.
Output side (s8f rank 2): ``fetch_audio`` (loudness normalisation, true-peak limiting, resampling to the client's rate and PCM16 / G.711 encoding of
the valid samples on the GPU + one pinned device->host copy), ``fetch_pcm16`` (the same at 16 kHz PCM16), ``pcm16_to_wav_bytes`` (the 16 kHz mono
PCM16 RIFF image the front-ends emit) and ``audio_to_wav_bytes`` (the same at any rate, and G.711).
"""
import struct
import threading
import time
from collections import namedtuple
from concurrent.futures import Future

import numpy as np
import torch

from . import audio

Request = namedtuple("Request", "speaker prompt phonemes content")


def load_symbol_table(path):
    """line -> index, exactly like inference_am_vocoder_joint.py:76-80 (tokenlist, speaker2)."""
    with open(path, encoding="utf-8") as f:
        return {t.strip(): idx for idx, t in enumerate(f.readlines())}


def parse_line(line):
    """``speaker|prompt|phonemes|content`` (inference_am_vocoder_joint.py:96-102).  Phonemes are
    whitespace separated; extra fields are ignored like the reference ignores them."""
    parts = line.strip().split("|")
    if len(parts) < 4:
        raise ValueError("expected <speaker>|<prompt>|<phoneme>|<content>, got %d field(s)" % len(parts))
    return Request(parts[0], parts[1], parts[2].split(), parts[3])


def encode(req, token2id, speaker2id):
    """-> (int64 ids, speaker id) or None for an unknown speaker (the reference skips such lines,
    inference_am_vocoder_joint.py:109-110).  An unknown phoneme raises KeyError like the reference (:113)."""
    if req.speaker not in speaker2id:
        return None
    ids = np.asarray([token2id[ph] for ph in req.phonemes], dtype=np.int64)
    if ids.size == 0:
        raise ValueError("empty phoneme sequence")
    return ids, int(speaker2id[req.speaker])


# ---- long text: phoneme lines cut into segments that are each an utterance of their own -----------------------------------

SOS_EOS = "<sos/eos>"           # the edge token every frontend line starts and ends with (frontend.py:28,57, frontend_cn.py:103,120)
# Break tokens the reference frontends emit.  Punctuation: frontend_cn.py:110-112 turns every punctuation mark into sp3,
# frontend_en.py:69-71 emits engsp4; sp4 and the English marks close sentences too.  Word and language boundaries: the rest.
PUNCTUATION_BREAKS = frozenset({"sp3", "sp4", "engsp4", ".", "?", "!"})
WORD_BREAKS = frozenset({"sp1", "sp2", "engsp1", "engsp2", "cn_eng_sp", "eng_cn_sp"})


def split_phonemes(phonemes, max_phonemes=256):
    """Cut a phoneme line (token strings, as ``parse_line`` yields them) into segments of at most ``max_phonemes`` tokens,
    each wrapped as ``<sos/eos> ... <sos/eos>`` like a frontend line, for ``JETSGenerator.forward(join=...)`` /
    ``MicroBatcher.submit_joined``.

    One leading and one trailing ``<sos/eos>`` are stripped; an inner ``<sos/eos>`` forces a cut and is dropped, so several
    frontend lines put together fall apart at their edges.  Greedily, a window of at most ``max_phonemes - 2`` inner tokens is
    cut after its last punctuation break (``PUNCTUATION_BREAKS``), else after its last word break (``WORD_BREAKS``), else at its
    end; the break token stays at the end of the left segment.  Joining the segments' inner tokens gives back the input's
    inner tokens (less the inner ``<sos/eos>``), and a wrapped line of at most ``max_phonemes`` tokens with no inner
    ``<sos/eos>`` comes back whole.  The default keeps every line of the reference's inference text whole (the longest has 223
    tokens).  Raises ValueError for ``max_phonemes < 3`` or an input with no inner token."""
    max_phonemes = int(max_phonemes)
    if max_phonemes < 3:
        raise ValueError("max_phonemes must be >= 3 (two <sos/eos> edges and one token), got %d" % max_phonemes)
    toks = list(phonemes)
    if toks and toks[0] == SOS_EOS:
        toks = toks[1:]
    if toks and toks[-1] == SOS_EOS:
        toks = toks[:-1]
    runs, cur = [], []
    for t in toks:
        if t != SOS_EOS:
            cur.append(t)
        elif cur:
            runs.append(cur)
            cur = []
    if cur:
        runs.append(cur)
    if not runs:
        raise ValueError("the phoneme line holds no token between its <sos/eos> edges")
    width = max_phonemes - 2
    segments = []
    for run in runs:
        i = 0
        while len(run) - i > width:
            window = run[i:i + width]
            cut = width                      # tokens the left segment keeps
            for breaks in (PUNCTUATION_BREAKS, WORD_BREAKS):
                at = [k for k, t in enumerate(window) if t in breaks]
                if at:
                    cut = at[-1] + 1
                    break
            segments.append(run[i:i + cut])
            i += cut
        segments.append(run[i:])
    return [[SOS_EOS] + s + [SOS_EOS] for s in segments]


NEUTRAL_CONTROLS = (1.0, 0.0, 1.0)      # (duration_scale, pitch_shift, energy_scale)


def speech_controls(speed=1.0, pitch_shift=0.0, energy_scale=1.0):
    """A serving API's ``speed`` (openaiapi.py:159) and the pitch / energy controls -> the per-item
    ``(duration_scale, pitch_shift, energy_scale)`` of ``JETSGenerator.forward``: duration_scale = 1 / speed, computed in
    double.  Raises ValueError for a non-finite or non-positive speed / energy_scale or a non-finite pitch_shift."""
    speed, pitch_shift, energy_scale = float(speed), float(pitch_shift), float(energy_scale)
    if not (np.isfinite(speed) and speed > 0):
        raise ValueError("speed must be finite and > 0, got %r" % speed)
    if not np.isfinite(pitch_shift):
        raise ValueError("pitch_shift must be finite, got %r" % pitch_shift)
    if not (np.isfinite(energy_scale) and energy_scale > 0):
        raise ValueError("energy_scale must be finite and > 0, got %r" % energy_scale)
    return (1.0 / speed, pitch_shift, energy_scale)


TOKEN_SPEED_RANGE = (1.0 / 16.0, 16.0)        # per-phoneme duration scales 1 / speed must lie in [1/16, 16] (modules.prosody_table)


def phoneme_controls(n, speed=1.0, pitch_shift=0.0, energy_scale=1.0):
    """``speech_controls`` where each control may also be a sequence of ``n`` values, one per phoneme.  Returns the
    ``(duration_scale, pitch_shift, energy_scale)`` triple with a float or a float64 array of length n in each place (an array
    only where one was given).  Per-phoneme speeds must lie in [1/16, 16].  Raises ValueError."""
    vals = []
    for name, v in (("speed", speed), ("pitch_shift", pitch_shift), ("energy_scale", energy_scale)):
        a = np.asarray(v, dtype=np.float64)
        if a.ndim > 1 or (a.ndim == 1 and a.shape[0] != n):
            raise ValueError("%s must be a float or a sequence of %d values (one per phoneme), got shape %s" % (name, n, a.shape))
        vals.append(a)
    sp, ps, es = vals
    if sp.ndim == ps.ndim == es.ndim == 0:
        return speech_controls(float(sp), float(ps), float(es))
    if not (np.all(np.isfinite(sp)) and np.all(sp > 0)):
        raise ValueError("speed must be finite and > 0")
    if sp.ndim == 1 and not (np.all(sp >= TOKEN_SPEED_RANGE[0]) and np.all(sp <= TOKEN_SPEED_RANGE[1])):
        raise ValueError("a per-phoneme speed must lie in [1/16, 16]")
    if not np.all(np.isfinite(ps)):
        raise ValueError("pitch_shift must be finite")
    if not (np.all(np.isfinite(es)) and np.all(es > 0)):
        raise ValueError("energy_scale must be finite and > 0")
    out = (1.0 / sp, ps, es)
    return tuple(float(x) if x.ndim == 0 else x for x in out)


GIVEN = ("durations", "pitch", "energy")


def given_values(n, durations=None, pitch=None, energy=None):
    """A request's caller-given ``durations`` (integer frames >= 0) / ``pitch`` / ``energy`` (finite) tracks, each None or a
    sequence of ``n`` values -> {name: int64 / float32 array} for the ones given.  Raises ValueError."""
    out = {}
    for name, v in (("durations", durations), ("pitch", pitch), ("energy", energy)):
        if v is None:
            continue
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        a = np.asarray(v)
        if a.shape != (n,):
            raise ValueError("%s must hold %d values (one per phoneme), got shape %s" % (name, n, a.shape))
        if name == "durations":
            if a.dtype.kind not in "iu" or (a.size and a.min() < 0):
                raise ValueError("durations must be integers >= 0")
            out[name] = a.astype(np.int64)
        else:
            if a.dtype.kind not in "fiu" or not np.all(np.isfinite(a)):
                raise ValueError("%s must be finite numbers" % name)
            out[name] = a.astype(np.float32)
    return out


def collate(items, device="cpu", pad_id=0):
    """items: list of (ids, speaker_id, style_vec, content_vec) -> the keyword arguments of
    ``JETSGenerator.forward`` (inference_am_vocoder_joint.py:113-128), padded with id 0 (the collate
    convention of the reference's dataset, prompt_dataset.py:183).

    An item may carry a fifth field, its ``(duration_scale, pitch_shift, energy_scale)`` (see ``speech_controls`` /
    ``phoneme_controls``).  When some item's controls are not neutral the result also holds the three controls: per-item
    lists, or (B,T) float64 tables when some item has per-phoneme values (each item's row holds its own values, per-item ones
    repeated along it; pads are neutral).  Otherwise it holds the five inputs only, so neutral traffic makes exactly the
    uncontrolled call.

    An item may carry a sixth field, the dict of ``given_values``.  Every item of the batch must then give the same tracks;
    they are padded to (B,T) with zeros (the padded entries are ignored by the model)."""
    B, T = len(items), max(len(it[0]) for it in items)
    ling = np.full((B, T), pad_id, dtype=np.int64)
    for b, it in enumerate(items):
        ling[b, :len(it[0])] = it[0]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)

    def vecs(col):
        # rows may be numpy arrays / lists, or tensors on any device (PromptEmbeddingCache.embed keeps them on the GPU)
        rows = [it[col] for it in items]
        if any(isinstance(r, torch.Tensor) for r in rows):
            return torch.stack([torch.as_tensor(r, dtype=torch.float32).to(device) for r in rows])
        return to(np.stack([np.asarray(r, dtype=np.float32) for r in rows]))

    out = dict(
        inputs_ling=to(ling),
        input_lengths=to(np.asarray([len(it[0]) for it in items], dtype=np.int64)),
        inputs_speaker=to(np.asarray([it[1] for it in items], dtype=np.int64)),
        inputs_style_embedding=vecs(2),
        inputs_content_embedding=vecs(3),
    )
    controls = [tuple(it[4]) if len(it) > 4 else NEUTRAL_CONTROLS for it in items]
    per_token = any(isinstance(x, np.ndarray) for c in controls for x in c)
    if per_token:
        for j, name in enumerate(("duration_scale", "pitch_shift", "energy_scale")):
            tab = np.full((B, T), NEUTRAL_CONTROLS[j], dtype=np.float64)
            for b, (it, c) in enumerate(zip(items, controls)):
                if isinstance(c[j], np.ndarray):
                    tab[b, :len(it[0])] = c[j]
                else:
                    tab[b, :] = c[j]            # a per-item value fills its whole row: the row is then one per-item scale
            out[name] = tab
    elif any(c != NEUTRAL_CONTROLS for c in controls):
        out["duration_scale"] = [c[0] for c in controls]
        out["pitch_shift"] = [c[1] for c in controls]
        out["energy_scale"] = [c[2] for c in controls]
    given = [it[5] if len(it) > 5 else {} for it in items]
    names = set(given[0])
    if any(set(g) != names for g in given):
        raise ValueError("every item of a batch must give the same caller tracks (durations / pitch / energy)")
    for name in sorted(names):
        tab = np.zeros((B, T), dtype=np.int64 if name == "durations" else np.float32)
        for b, (it, g) in enumerate(zip(items, given)):
            tab[b, :len(it[0])] = g[name]
        out[name] = to(tab)
    return out


class MicroBatcher:
    """Groups concurrent synthesis requests into padded batches.

    ``forward(**kwargs) -> dict`` is the model (``emotivoice_b200.modules.JETSGenerator``); requests are
    ``(ids, speaker_id, style_vec, content_vec)``.  ``submit`` returns a Future whose result is the item's
    float32 waveform trimmed to its own length (``mel_lengths[b] * hop``).  A worker thread collects up to
    ``max_batch`` requests, waiting at most ``max_wait_s`` after the first one, and runs ONE forward.
    Errors of a batch are delivered to every future of that batch.  Requests with different prosody controls
    (``speed``, ``pitch_shift``, ``energy_scale``, per item or per phoneme) share one forward.  Requests that give their
    own ``durations`` / ``pitch`` / ``energy`` run in one forward with the requests that give the same set of tracks.

    ``submit_joined`` takes a long text as segments (``split_phonemes``): they enter a forward as consecutive items of one
    ``join`` group, so the text comes back as one waveform; plain requests of that forward each get a group of their own.
    ``max_batch`` counts items.  A joined request is never split across forwards; one with more segments than ``max_batch``
    runs alone.  A forward without a joined request is called exactly as before, with no ``join`` keyword.

    A request that gives ``sample_rate``, ``encoding``, ``loudness`` and / or ``true_peak`` gets a numpy array in that format
    instead (``fetch_audio``; the model then needs ``format_audio``).  Requests in different formats share a forward: one output
    launch set (a loudness measurement for a ``loudness`` target, the limiter's passes for a ``true_peak`` ceiling) and one copy
    per distinct format.
    """

    def __init__(self, forward, device="cpu", max_batch=32, max_wait_s=0.005, hop=256):
        self._forward, self._device, self._hop = forward, device, hop
        self._sr = int(getattr(getattr(forward, "config", None), "sr", 16000))
        self._max_batch, self._max_wait = int(max_batch), float(max_wait_s)
        self._lock = threading.Condition()
        self._queue = []
        self._closed = False
        self.batches_run = 0
        self._thread = threading.Thread(target=self._loop, name="ev-microbatcher", daemon=True)
        self._thread.start()

    def submit(self, ids, speaker_id, style_vec, content_vec, speed=1.0, pitch_shift=0.0, energy_scale=1.0, durations=None,
               pitch=None, energy=None, sample_rate=None, encoding=None, loudness=None, true_peak=None, watermark=None):
        """``speed`` > 1 speaks faster (duration_scale = 1 / speed); ``pitch_shift`` in semitones; ``energy_scale``
        multiplies frame energy.  Each is a float or a sequence of ``len(ids)`` values, one per phoneme (a per-phoneme speed
        must lie in [1/16, 16]).  ``durations`` (integer frames), ``pitch`` and ``energy`` (the predictors' normalised units):
        None or ``len(ids)`` values that replace the model's predictions (see ``JETSGenerator.forward``).  ``sample_rate`` /
        ``encoding`` / ``loudness`` / ``true_peak`` / ``watermark``: see ``_output_format``.  Invalid values raise ValueError here, so they cannot
        fail a batch of other requests."""
        ids = np.asarray(ids, dtype=np.int64)
        controls = phoneme_controls(len(ids), speed, pitch_shift, energy_scale)
        given = given_values(len(ids), durations, pitch, energy)
        fmt = self._output_format(sample_rate, encoding, loudness, true_peak, watermark)
        item = (ids, int(speaker_id), style_vec, content_vec, controls) + ((given,) if given else ())
        return self._enqueue([item], False, fmt)

    def submit_joined(self, segments, speaker_id, style_vec, content_vec, speed=1.0, pitch_shift=0.0, energy_scale=1.0,
                      sample_rate=None, encoding=None, loudness=None, true_peak=None, watermark=None):
        """One long text as ``segments``: a list of phoneme id arrays, e.g. ``split_phonemes`` output put through ``encode``.
        ``style_vec`` / ``content_vec``: one vector for every segment, or a list (or a 2-D array) with one vector per segment,
        for a different prompt per sentence.  ``speed`` / ``pitch_shift`` / ``energy_scale``: one float each, checked as in
        ``submit``.  The future's result is the text's float32 waveform, the segments' mel joined and vocoded as one,
        trimmed to ``joined_lengths[g] * hop``, or that waveform in the format of ``sample_rate`` / ``encoding`` / ``loudness`` /
        ``true_peak`` / ``watermark`` (see ``_output_format``).  Raises ValueError here for invalid arguments."""
        segs = [np.asarray(s, dtype=np.int64) for s in segments]
        if not segs or any(s.ndim != 1 or s.size == 0 for s in segs):
            raise ValueError("segments must be a non-empty list of non-empty 1-D phoneme id arrays")
        controls = speech_controls(speed, pitch_shift, energy_scale)
        styles = _per_segment("style_vec", style_vec, len(segs))
        contents = _per_segment("content_vec", content_vec, len(segs))
        fmt = self._output_format(sample_rate, encoding, loudness, true_peak, watermark)
        items = [(s, int(speaker_id), st, ct, controls) for s, st, ct in zip(segs, styles, contents)]
        return self._enqueue(items, True, fmt)

    def _output_format(self, sample_rate, encoding, loudness, true_peak=None, watermark=None):
        """A request's output format: None when all five are None (the result is the float32 waveform tensor, as always), else
        the ``audio.OutputFormat`` ``fetch_audio`` is called with: the result is then a numpy array at ``sample_rate`` (None: the
        model's rate) in ``encoding`` (None: "pcm16"), normalised to ``loudness`` LUFS (None: not normalised), limited to
        ``true_peak`` dBTP (None: not limited) and marked with the key ``watermark`` (None: not marked).  Requests with different
        keys have different formats, so each key gets its own ``fetch_audio`` call.  Raises ValueError for a rate, encoding,
        loudness target, ceiling or key ``format_audio`` does not take."""
        if sample_rate is None and encoding is None and loudness is None and true_peak is None and watermark is None:
            return None
        return audio.output_format(sample_rate, "pcm16" if encoding is None else encoding, loudness, true_peak, self._sr,
                                   watermark=watermark)

    def _enqueue(self, items, joined, fmt):
        fut = Future()
        with self._lock:
            if self._closed:
                raise RuntimeError("MicroBatcher is closed")
            self._queue.append((items, fut, joined, fmt))
            self._lock.notify()
        return fut

    def close(self):
        with self._lock:
            self._closed = True
            self._lock.notify()
        self._thread.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _take(self):
        with self._lock:
            while not self._queue and not self._closed:
                self._lock.wait()
            if not self._queue:
                return None
            deadline = time.monotonic() + self._max_wait
            while sum(len(e[0]) for e in self._queue) < self._max_batch and not self._closed:
                left = deadline - time.monotonic()
                if left <= 0:
                    break
                self._lock.wait(left)
            n = items = 0                    # whole requests in arrival order up to max_batch items; the first one always
            while n < len(self._queue) and (n == 0 or items + len(self._queue[n][0]) <= self._max_batch):
                items += len(self._queue[n][0])
                n += 1
            batch, self._queue = self._queue[:n], self._queue[n:]
            return batch

    def _loop(self):
        while True:
            batch = self._take()
            if batch is None:
                return
            groups = {}                      # one forward per set of caller-given tracks (the common case: one group)
            for entry in batch:
                it = entry[0][0]
                groups.setdefault(tuple(sorted(it[5])) if len(it) > 5 else (), []).append(entry)
            for group in groups.values():
                self._run(group)

    def _run(self, batch):
        futs = [e[1] for e in batch]
        try:
            kw = collate([it for e in batch for it in e[0]], self._device)
            joined = any(e[2] for e in batch)
            if joined:                       # one group per request: a joined request's segments share its id
                kw["join"] = [g for g, e in enumerate(batch) for _ in e[0]]
            out = self._forward(**kw)
            # request r's output is item r of the forward (group r of a joined one); one format_audio call and one copy
            # per distinct OutputFormat, over the requests that asked for it
            formats = {}
            for r, e in enumerate(batch):
                if e[3] is not None:
                    formats.setdefault(e[3], []).append(r)
            results = {}
            for f, rs in formats.items():
                mark = {} if f.watermark is None else {"watermark": f.watermark}     # only asked of fetch_audio when used
                results.update(zip(rs, fetch_audio(self._forward, out, f.rate, f.encoding, items=rs, hop=self._hop, loudness=f.loudness,
                                                   true_peak=f.true_peak, **mark)))
            if len(results) < len(batch):
                wav = out["wav_predictions"]
                lens = out.get("joined_lengths_host", out.get("joined_lengths")) if joined else out.get("mel_lengths")
                lens = [int(wav.shape[-1]) // self._hop] * len(batch) if lens is None else [int(v) for v in lens.tolist()]
                wav = wav.detach().cpu()
                for b in range(len(batch)):
                    if b not in results:
                        results[b] = wav[b, 0, :lens[b] * self._hop].clone()
            self.batches_run += 1
            for b, f in enumerate(futs):
                f.set_result(results[b])
        except BaseException as e:       # deliver, keep serving
            for f in futs:
                if not f.done():
                    f.set_exception(e)


def _per_segment(name, v, n):
    """``submit_joined``'s style / content argument -> n vectors: one vector repeated, or a list / 2-D array of n vectors."""
    if isinstance(v, (list, tuple)) and len(v) and (getattr(v[0], "ndim", 0) >= 1 or isinstance(v[0], (list, tuple))):
        rows = list(v)
    elif getattr(v, "ndim", 1) == 2:
        rows = [v[i] for i in range(v.shape[0])]
    else:
        return [v] * n
    if len(rows) != n:
        raise ValueError("%s holds %d vectors for %d segments" % (name, len(rows), n))
    return rows


# ---- output side (SURVEY.md s8f rank 2): the on-wire format every front-end emits -----------------------------------

def pcm16_to_wav_bytes(pcm, sample_rate=16000):
    """int16 mono samples -> a complete RIFF/WAVE file image (PCM, 16 bit, mono), i.e. what the reference writes with
    ``sf.write(path, int16_audio, samplerate=config.sampling_rate)`` (inference_am_vocoder_joint.py:132-134) and what
    openaiapi.py:139-140,172-174 sends for ``response_format="wav"``.  44-byte canonical header, little endian."""
    pcm = np.ascontiguousarray(np.asarray(pcm))
    if pcm.dtype != np.int16 or pcm.ndim != 1:
        raise ValueError("expected a 1-D int16 array, got %s %s" % (pcm.dtype, pcm.shape))
    data = pcm.astype("<i2", copy=False).tobytes()
    if len(data) > 0xFFFFFFFF - 36:
        raise ValueError("waveform too long for a RIFF container")
    header = struct.pack("<4sI4s4sIHHIIHH4sI", b"RIFF", 36 + len(data), b"WAVE", b"fmt ", 16,
                         1, 1, int(sample_rate), int(sample_rate) * 2, 2, 16, b"data", len(data))
    return header + data


WAV_G711_TAGS = {"mulaw": 7, "alaw": 6}       # WAVE_FORMAT_MULAW / WAVE_FORMAT_ALAW


def audio_to_wav_bytes(samples, sample_rate, encoding="pcm16"):
    """Samples as ``fetch_audio`` returns them -> a complete mono RIFF/WAVE file image.  "pcm16": ``pcm16_to_wav_bytes``.
    "mulaw" / "alaw" (uint8 G.711 codes): format tag 7 / 6, 8 bits, an 18-byte ``fmt `` chunk with cbSize = 0 and a ``fact``
    chunk holding the sample count, as non-PCM WAVE files carry them; a pad byte follows odd-length data."""
    if encoding == "pcm16":
        return pcm16_to_wav_bytes(samples, sample_rate)
    if encoding not in WAV_G711_TAGS:
        raise ValueError("a WAV image holds pcm16, mulaw or alaw samples, got %r" % (encoding,))
    codes = np.ascontiguousarray(np.asarray(samples))
    if codes.dtype != np.uint8 or codes.ndim != 1:
        raise ValueError("expected a 1-D uint8 array of G.711 codes, got %s %s" % (codes.dtype, codes.shape))
    data = codes.tobytes()
    pad = len(data) & 1
    if len(data) + pad > 0xFFFFFFFF - 50:
        raise ValueError("waveform too long for a RIFF container")
    rate = int(sample_rate)
    header = struct.pack("<4sI4s4sIHHIIHHH4sII4sI", b"RIFF", 50 + len(data) + pad, b"WAVE", b"fmt ", 18,
                         WAV_G711_TAGS[encoding], 1, rate, rate, 1, 8, 0, b"fact", 4, len(data), b"data", len(data))
    return header + data + b"\0" * pad


def fetch_audio(model, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None,
                watermark=None):
    """Finish one forward in the format a client asked for: ``model.format_audio`` resamples to ``sample_rate`` (None: the
    model's 16 kHz) and encodes ("float32", "pcm16", "mulaw" or "alaw") only the valid samples of each output, packed, on the
    GPU, after normalising each output to ``loudness`` LUFS when that is given (BS.1770-4 integrated loudness, -1 dBFS
    sample-peak ceiling; see ``format_audio``) and limiting each to ``true_peak`` dBTP when that is given (a look-ahead
    true-peak limiter, which replaces the sample-peak ceiling), each marked with the key ``watermark`` when that is given
    (``emotivoice_b200.watermark.detect`` finds the mark); then ONE device->host copy of that buffer into pinned memory.  ``out`` is the
    dict ``model(...)`` returned; ``items`` selects outputs (default: all).  Returns a list of 1-D numpy arrays (float32, int16
    or uint8), one per batch item, or per group of a joined forward.  "flac": each array is the bytes of a complete .flac file
    whose samples are the "pcm16" result.  Invalid arguments raise ValueError before anything is enqueued."""
    packed, offs = model.format_audio(out, sample_rate, encoding, items=items, hop=hop, loudness=loudness, true_peak=true_peak,
                                      watermark=watermark)
    host = torch.empty(packed.shape, dtype=packed.dtype, pin_memory=True)
    host.copy_(packed, non_blocking=True)
    torch.cuda.current_stream(packed.device).synchronize()
    arr = host.numpy()
    return [arr[offs[k]:offs[k + 1]].copy() for k in range(len(offs) - 1)]


def fetch_pcm16(model, out, hop=256):
    """Finish one forward the way the callers do (inference_am_vocoder_joint.py:130-131), without the fp32 waveform
    ever crossing PCIe: ``wav * 32768 -> int16`` on the GPU (saturating, see ``model.to_pcm16``) for the samples up to
    ``mel_lengths[b] * hop`` (``joined_lengths_host[g] * hop`` for the output of a joined forward), then ONE device->host copy
    into pinned memory: ``fetch_audio`` at the model's rate.  Returns a list of 1-D int16 numpy arrays (one per batch item, or
    per group of a joined forward)."""
    return fetch_audio(model, out, hop=hop)


# ---- prompt / content embeddings (SURVEY.md s8f rank 1: "batched, prompt-embedding cache") -----------------------------

class PromptEmbeddingCache:
    """The callers' ``get_style_embedding`` (inference_am_vocoder_joint.py:25-38) for many texts at once, with a cache.

    The reference tokenises ONE text and runs the BERT style encoder on the CPU, twice per utterance (prompt and content,
    :106-107), recomputing identical prompts ("Happy", "Sad", ... repeat for every line).  Here all texts of a call that are
    not cached go through the tokenizer as one right-padded batch and through ``style_encoder`` as ONE forward; results are
    kept (LRU, on the encoder's device) keyed by the text.  Batching is invisible: the engine's padded batches are bitwise
    equal to single-item calls.

    ``tokenizer(list_of_str, return_tensors="pt", padding=True)`` -> dict with input_ids / token_type_ids / attention_mask
    (a transformers tokenizer, as in the reference); ``style_encoder(**those)`` -> dict with "pooled_output" (B, 768)
    (``emotivoice_b200.style.StyleEncoder`` or the reference's own module).
    """

    def __init__(self, tokenizer, style_encoder, device=None, max_entries=4096):
        from collections import OrderedDict
        self._tok, self._enc, self._device = tokenizer, style_encoder, device
        self._max = int(max_entries)
        self._cache = OrderedDict()
        self._lock = threading.Lock()
        self.hits = self.misses = self.forwards = 0

    def embed(self, texts):
        """list of str -> (len(texts), D) float32 tensor, row i = pooled_output of texts[i]."""
        texts = list(texts)
        uniq = list(dict.fromkeys(texts))
        have = {}
        # rows are captured into a local dict inside the critical section that finds them, so a concurrent embed() that evicts
        # them afterwards cannot make this call's final lookup fail
        with self._lock:
            for t in uniq:
                row = self._cache.get(t)
                if row is not None:
                    self._cache.move_to_end(t)
                    have[t] = row
            n_hit = sum(1 for t in texts if t in have)
            self.hits += n_hit
            self.misses += len(texts) - n_hit
        missing = [t for t in uniq if t not in have]
        if missing:
            enc = self._tok(missing, return_tensors="pt", padding=True)
            keys = ("input_ids", "token_type_ids", "attention_mask")
            args = {k: (enc[k].to(self._device) if self._device is not None else enc[k]) for k in keys}
            with torch.no_grad():
                pooled = self._enc(**args)["pooled_output"].detach()
            fresh = {t: pooled[i].clone() for i, t in enumerate(missing)}
            have.update(fresh)
            with self._lock:
                self.forwards += 1
                self._cache.update(fresh)
                while len(self._cache) > self._max:
                    self._cache.popitem(last=False)
        return torch.stack([have[t] for t in texts])
