"""Host-side mirror of the reference's model boundary (SURVEY.md s8b).

Same class names, constructor arguments, ``state_dict`` keys, ``forward()`` keyword
signature and returned dict as

* ``JETSGenerator``  -- models/prompt_tts_modified/jets.py:26-71
* ``PromptTTS``      -- models/prompt_tts_modified/model_open_source.py:14-163
* ``Generator``      -- models/hifigan/models.py:90-140

so the reference's callers (inference_am_vocoder_joint.py:70-74,120-129, demo_page.py:88-92,
openaiapi.py:78-82) run unchanged: ``JETSGenerator(conf).to(device)``,
``.load_state_dict(torch.load(path)['generator'])``, ``.eval()``, call under ``no_grad``.

The modules hold ``nn.Parameter`` trees only (for state-dict compatibility); every FLOP
of ``forward`` runs in libemotivoice_b200.so (hand-written sm_90a kernels) through the C
ABI in include/emotivoice_b200.h.  PyTorch provides device memory and the stream.  There
is no CPU path: calling ``forward`` on CPU tensors raises.
"""
import ctypes
import functools
import threading

import numpy as np
import torch
import torch.nn as nn

from . import _abi, audio, output, packing, synth
from .loudness import check_rate as check_meter_rate


class _Holder(nn.Module):
    """Parameter container; never called."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: compute happens in libemotivoice_b200.so")


_TLS = threading.local()          # per-thread pinned read-back buffer + event


# Statistics of the pitch / energy targets the predictors were trained on (config.pitch_stats / energy_stats of the reference,
# config/joint/config.py:108,111; prompt_dataset.py:130-142 normalises as (x - mean) / std).  Used when the config has none.
PITCH_STATS = (225.089, 53.78)
ENERGY_STATS = (30.610, 21.78)


def _per_item(name, v, B, neutral, T=None):
    """None / float / length-B sequence / CPU tensor -> float64 numpy (B,); with T given also a (B,T) nested sequence or CPU
    tensor -> (B,T).  Raises ValueError before anything is enqueued."""
    if v is None:
        return np.full(B, neutral, dtype=np.float64)
    if isinstance(v, torch.Tensor):
        if v.device.type != "cpu":
            raise ValueError("%s must be a float, a sequence or a CPU tensor (reading a %s tensor would synchronise the device)"
                             % (name, v.device.type))
        v = v.detach().double().numpy()
    try:
        a = np.asarray(v, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError("%s must be a float, a length-%d sequence or a CPU tensor" % (name, B)) from None
    if a.ndim == 0:
        return np.full(B, float(a), dtype=np.float64)
    if a.shape != (B,) and (T is None or a.shape != (B, T)):
        raise ValueError("%s has shape %s, expected a float, length %d%s" % (name, a.shape, B, "" if T is None else " or (%d, %d)" % (B, T)))
    return a


# Per-token duration scales are kept in this range: every fp32 value >= 1/16 is a multiple of 2^-27, which keeps the duration scan's
# fp64 sums exact whatever the mix of scales in an utterance (see duration_scan_kernel).  Per-item scales, and rows of a (B,T) table
# that hold one value throughout, only need to be > 0.
TOKEN_SCALE_RANGE = (1.0 / 16.0, 16.0)


def prosody_table(B, duration_scale=None, pitch_shift=None, energy_scale=None, config=None, T=None):
    """Host side of the prosody controls: -> None when every item is neutral, else a float32 CPU tensor of rows
    {alpha, p_scale, p_shift, e_scale, e_shift}: (B,5) with one row per item, or (B,T,5) with one row per token when T is given
    and some control is a (B,T) table (the per-item ones are then repeated along T).  alpha = fl32(duration_scale)
    (GaussianUpsampling's alpha, alignment.py:183); with r = 2^(semitones/12): p_scale = fl32(r), p_shift = fl32(mean (r-1) / std)
    in the normalised units of the pitch predictor, so that the shifted track is the normalised pitch of r * f0; energy likewise
    with r = energy_scale.  A (B,T) duration_scale must lie in [1/16, 16], except in rows that hold one value throughout."""
    a = _per_item("duration_scale", duration_scale, B, 1.0, T)
    s = _per_item("pitch_shift", pitch_shift, B, 0.0, T)
    e = _per_item("energy_scale", energy_scale, B, 1.0, T)
    if not (np.all(np.isfinite(a)) and np.all(a > 0)):
        raise ValueError("duration_scale must be finite and > 0, got %s" % a.tolist())
    if not np.all(np.isfinite(s)):
        raise ValueError("pitch_shift must be finite, got %s" % s.tolist())
    if not (np.all(np.isfinite(e)) and np.all(e > 0)):
        raise ValueError("energy_scale must be finite and > 0, got %s" % e.tolist())
    if a.ndim == 2:                 # a row with one value throughout is a per-item scale and keeps the per-item range
        a32 = a.astype(np.float32)
        lo, hi = TOKEN_SCALE_RANGE
        varies = np.any(a32 != a32[:, :1], axis=1, keepdims=True)
        if np.any(varies & ((a32 < lo) | (a32 > hi))):
            raise ValueError("a per-token duration_scale must lie in [1/16, 16] (a row with one value throughout may hold any "
                             "scale > 0), got values in [%g, %g]" % (a.min(), a.max()))
    if np.all(a == 1.0) and np.all(s == 0.0) and np.all(e == 1.0):
        return None
    if max(a.ndim, s.ndim, e.ndim) == 2:
        a, s, e = (np.broadcast_to(x if x.ndim == 2 else x[:, None], (B, T)) for x in (a, s, e))
    mp, sp = getattr(config, "pitch_stats", None) or PITCH_STATS
    me, se = getattr(config, "energy_stats", None) or ENERGY_STATS
    with np.errstate(over="ignore", invalid="ignore"):
        rp = np.exp2(s / 12.0)
        tab = np.stack([a, rp, float(mp) * (rp - 1.0) / float(sp), e, float(me) * (e - 1.0) / float(se)], axis=-1)
        tab32 = np.ascontiguousarray(tab.astype(np.float32))
    if not (np.all(np.isfinite(tab32)) and np.all(tab32[..., 0] > 0) and np.all(tab32[..., 3] > 0)):
        raise ValueError("prosody controls outside the fp32 range: duration_scale %s, pitch_shift %s, energy_scale %s"
                         % (a.tolist(), s.tolist(), e.tolist()))
    return torch.from_numpy(tab32)


def caller_values(name, v, B, T, device, integer):
    """A caller-given ``durations`` (integer) or ``pitch`` / ``energy`` (float) track -> None, a (B,T) int64 / float32 CPU tensor
    (validated here: durations >= 0, tracks finite), or a (B,T) tensor on ``device`` (taken as it is: int64 / float32 exactly,
    since converting it would enqueue work).  (T,) is accepted when B == 1, so that the squeezed predictions of a forward can
    be passed straight back.  Raises ValueError before anything is enqueued."""
    if v is None:
        return None
    want = torch.int64 if integer else torch.float32
    kind = "an integer" if integer else "a floating-point"
    if isinstance(v, torch.Tensor) and v.device.type != "cpu":
        if v.device != torch.device(device):
            raise ValueError("%s is on %s but the module is on %s" % (name, v.device, device))
        if v.dtype != want:
            raise ValueError("%s on the device must be %s, got %s" % (name, want, v.dtype))
        t = v.detach()
    else:
        a = v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        if a.dtype.kind not in (("i", "u") if integer else ("f",)) and not (a.dtype == object and a.size == 0):
            raise ValueError("%s must hold %s type, got %s" % (name, kind, a.dtype))
        if integer:
            if a.size and (a.min() < 0):
                raise ValueError("%s must be >= 0 (frames per phoneme), got a minimum of %d" % (name, int(a.min())))
            if a.size and a.max() > np.iinfo(np.int64).max:
                raise ValueError("%s holds values beyond the int64 range" % name)
        elif not np.all(np.isfinite(a)):
            raise ValueError("%s must be finite" % name)
        t = torch.from_numpy(np.ascontiguousarray(a.astype(np.int64 if integer else np.float32)))
    if tuple(t.shape) != (B, T) and not (B == 1 and t.numel() == T and t.dim() <= 1):
        raise ValueError("%s has shape %s, expected (%d, %d)%s" % (name, tuple(t.shape), B, T, " or (%d,)" % T if B == 1 else ""))
    return t.reshape(B, T).contiguous()


def controls_for(module, inputs_ling, duration_scale, pitch_shift, energy_scale, durations, pitch, energy):
    """Every host-side check of the controls of ``forward``, before anything is packed or enqueued -> (prosody table or None,
    {"durations": .., "pitch": .., "energy": ..} with None for an absent one)."""
    B, T = int(inputs_ling.shape[0]), int(inputs_ling.shape[1])
    prosody = prosody_table(B, duration_scale, pitch_shift, energy_scale, module.config, T=T)
    dev = next(module.parameters()).device
    given = dict(durations=caller_values("durations", durations, B, T, dev, True),
                 pitch=caller_values("pitch", pitch, B, T, dev, False),
                 energy=caller_values("energy", energy, B, T, dev, False))
    return prosody, given


JOIN_MAX_ITEMS = 4096             # items of one joined forward: ev_join_mel keeps their offsets in shared memory


def join_groups(join, B):
    """The ``join`` of ``forward`` -> None, or the (B,) int32 numpy group ids: a sequence or CPU tensor of B integers, 0 first,
    each next one equal to the previous one or one more.  Raises ValueError before anything is enqueued."""
    if join is None:
        return None
    if isinstance(join, torch.Tensor):
        if join.device.type != "cpu":
            raise ValueError("join must be a sequence or a CPU tensor (reading a %s tensor would synchronise the device)"
                             % join.device.type)
        join = join.detach().numpy()
    try:
        a = np.asarray(join)
    except (TypeError, ValueError):
        raise ValueError("join must hold %d integer group ids" % B) from None
    if a.shape != (B,) or a.dtype.kind not in "iu":
        raise ValueError("join must hold %d integer group ids (one per batch item), got %s of shape %s" % (B, a.dtype, a.shape))
    if B > JOIN_MAX_ITEMS:
        raise ValueError("a joined forward takes at most %d items, got %d" % (JOIN_MAX_ITEMS, B))
    steps = np.diff(a.astype(np.int64))
    if a[0] != 0 or np.any((steps != 0) & (steps != 1)):
        raise ValueError("join must start at 0 and each next id must equal the previous one or one more, got %s" % a.tolist())
    return a.astype(np.int32)


def group_frames(group, mel_lens_host):
    """(B,) group ids and per-item frame counts -> (G,) int64 frames of each joined output."""
    out = np.zeros(int(group[-1]) + 1, dtype=np.int64)
    np.add.at(out, group, np.asarray(mel_lens_host, dtype=np.int64))
    return out


def _bucket(nbytes):
    """Workspace sizes are rounded up to a geometric series (x1.125 steps, 2 MiB granularity): utterances of similar length
    then request IDENTICAL sizes, so torch's caching allocator serves them from its pool instead of calling cudaMalloc
    (a device-synchronising, ~1-2 ms call) whenever a request is a little larger than anything it has cached."""
    g = 2 << 20
    n = max(int(nbytes), g)
    b = g
    while b < n:
        b = (b + (b >> 3) + g - 1) // g * g
    return b


def _workspace(arena, device, kind, nbytes):
    """Grow-only workspace arena ``arena``: (stream, kind) -> uint8 buffer: after the largest request has been seen (or
    `reserve`d) no call allocates device memory any more -- a fresh cudaMalloc in the middle of a forward is a
    device-synchronising stall of milliseconds.  Reuse across calls is safe because every use is ordered on the stream the
    buffer belongs to."""
    key = (torch.cuda.current_stream(device).cuda_stream, kind)
    t = arena.get(key)
    if t is None or t.numel() < nbytes:
        arena.pop(key, None)
        t = None
        t = torch.empty((_bucket(nbytes),), dtype=torch.uint8, device=device)
        arena[key] = t
    return t


def _register(root, dotted, tensor):
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Holder())
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


def _legacy_weight_norm_hook(module, state_dict, prefix, *args):
    """Checkpoints written by torch < 2.1 carry weight_g / weight_v instead of
    parametrizations.weight.original0/1 (SURVEY.md s5, checkpoint row): accept both."""
    for k in list(state_dict.keys()):
        if not k.startswith(prefix):
            continue
        if k.endswith(".weight_g"):
            state_dict[k[:-len("weight_g")] + "parametrizations.weight.original0"] = state_dict.pop(k)
        elif k.endswith(".weight_v"):
            state_dict[k[:-len("weight_v")] + "parametrizations.weight.original1"] = state_dict.pop(k)


def _dirty_post_hook(module, incompatible_keys):
    for m in module.modules():
        if isinstance(m, _EngineOwner):
            m._ev_dirty = True


class _Engine:
    """One ev_ctx + its packed weight blob and positional table on one device."""

    def __init__(self, conf, packed, device, precision="fp32", blob=None, index_meta=None):
        """``packed``: name -> tensor dict (packing.pack_state_dict + add_tc_weights), laid into one blob here; or pass a
        ready ``blob`` (fp32 tensor already on ``device``) with its ``index_meta`` [(name, offset, numel)] -- what the
        other ranks of a multi-GPU run receive from rank 0 instead of re-packing (runner.broadcast_engine)."""
        self.lib = _abi.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("emotivoice_b200 runs on CUDA (sm_90a) only; got device %s. "
                               "There is no CPU fallback." % (self.device,))
        self.index_dev = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.cfg = _abi.make_config(conf)
        self.hidden = int(self.cfg.hidden)
        handle = ctypes.c_void_p()
        _abi.check(self.lib.ev_create(ctypes.byref(handle), self.index_dev, ctypes.byref(self.cfg)))
        self.handle = handle
        if blob is None:
            blob, self.index = packing.make_blob(packed)
            self.blob = blob.to(self.device)
        else:
            self.index = packing.index_from_meta(index_meta)
            self.blob = blob
            assert blob.device == self.device and blob.dtype == torch.float32 and blob.is_contiguous()
        self.set_precision(precision)         # first: binding checks that the blob carries the weight copies this precision reads
        _abi.check(self.lib.ev_bind_weights(self.handle, self.blob.data_ptr(), self.blob.numel(),
                                            ctypes.cast(self.index, ctypes.c_void_p), len(self.index)))
        self.pe = None
        # the arena does not refer back to the engine, so the output chain can hold it without a reference cycle
        self._ws = functools.partial(_workspace, {}, self.device)
        self.call_lock = threading.RLock()      # one forward at a time enqueues on an engine (its workspaces are reused, stream-ordered)
        self.output = output.Chain(self.device, self.lib, self._ws)
        self.ensure_pe(5000)          # PositionalEncoding max_len=5000 (encoder.py:206)
        self.total_up = int(np.prod([self.cfg.up_rates[i] for i in range(self.cfg.n_ups)]))

    def set_precision(self, precision):
        _abi.check(self.lib.ev_set_precision(self.handle, _abi.PRECISIONS[precision]))
        self.precision = precision

    def index_meta(self):
        return [(e.name.decode(), int(e.offset), int(e.numel)) for e in self.index]

    def ensure_pe(self, n):
        if self.pe is not None and self.pe.shape[0] >= n:
            return
        n = max(n, 2 * (self.pe.shape[0] if self.pe is not None else 0))
        self.pe = packing.build_pe_table(n, self.hidden).to(self.device)
        _abi.check(self.lib.ev_bind_pe(self.handle, self.pe.data_ptr(), n))

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.ev_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # -- calls ------------------------------------------------------------------------
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def reserve(self, batch, phonemes, frames):
        """Pre-size the arena of the current stream for requests up to (batch, phonemes, frames)."""
        lib = self.lib
        fs = {int(frames)}
        if batch * frames > 2400:                 # small batches carry extra grouped-launch buffers: cover the largest of those shapes too
            fs.add(max(1, 2400 // int(batch)))
        with self.call_lock:
            self.ensure_pe(max(int(frames), int(phonemes)))
            self._ws("p1", lib.ev_phase1_workspace_bytes(self.handle, int(batch), int(phonemes)))
            self._ws("p2", max(lib.ev_phase2_workspace_bytes(self.handle, int(batch), f) for f in fs))

    def _read_back(self, t):
        """Device int32 vector -> host tensor, waiting by polling."""
        tl = _TLS
        n = t.numel()
        if getattr(tl, "pin", None) is None or tl.pin.numel() < n:
            tl.pin = torch.empty((max(n, 1024),), dtype=torch.int32).pin_memory()
            tl.ev = torch.cuda.Event()
        tl.pin[:n].copy_(t, non_blocking=True)
        tl.ev.record(torch.cuda.current_stream(self.device))
        while not tl.ev.query():
            pass
        return tl.pin[:n].clone()

    def acoustic(self, ling, lens, spk, style, content, invariant, prosody=None, given=None, group=None):
        """``prosody``: None (neutral: the plain ev_am_phase1 call) or the (B,5) / (B,T,5) CPU table of ``prosody_table``;
        ``given``: None or the caller's {"durations", "pitch", "energy"} of ``controls_for`` (each None, a CPU or a device tensor);
        ``group``: None or the (B,) int32 group ids of ``join_groups`` (a joined forward: the result then also carries the group
        ids on the device, the group lengths on the host and on the device, and a phase-2 workspace the joined vocoder pass fits)."""
        lib, dev = self.lib, self.device
        B, T = ling.shape
        self.ensure_pe(T)
        pinned = []                   # CPU sources are uploaded with the inputs; the pinned copies live until the read-back below

        def upload(t):
            if t is None or t.device == dev:
                return t
            pinned.append(t.pin_memory())
            return pinned[-1].to(dev, non_blocking=True)
        prosody = upload(prosody)
        given = {k: upload(v) for k, v in (given or {}).items()}
        group_dev = None if group is None else upload(torch.from_numpy(group))
        caller = {k: v for k, v in given.items() if v is not None}
        dur = torch.empty((B, T), dtype=torch.int64, device=dev)
        pitch = torch.empty((B, T), dtype=torch.float32, device=dev)
        energy = torch.empty((B, T), dtype=torch.float32, device=dev)
        meta = torch.empty((2 * B + 2,), dtype=torch.int32, device=dev)      # lens32 (B) | mel_lens (B) | max | input status
        ws1 = self._ws("p1", lib.ev_phase1_workspace_bytes(self.handle, B, T))
        n1 = ws1.numel()
        st = self._stream()
        lens32_ptr = meta.data_ptr()
        mel_lens_ptr = meta.data_ptr() + 4 * B
        ptr = lambda t: None if t is None else t.data_ptr()
        if caller or (prosody is not None and prosody.dim() == 3):
            _abi.check(lib.ev_am_phase1_controls(self.handle, ling.data_ptr(), lens.data_ptr(), spk.data_ptr(), style.data_ptr(),
                                                 content.data_ptr(), B, T, int(invariant), ptr(prosody),
                                                 int(prosody is not None and prosody.dim() == 3), ptr(given.get("durations")),
                                                 ptr(given.get("pitch")), ptr(given.get("energy")), dur.data_ptr(), pitch.data_ptr(),
                                                 energy.data_ptr(), lens32_ptr, mel_lens_ptr, ws1.data_ptr(), n1, st))
        elif prosody is None:
            _abi.check(lib.ev_am_phase1(self.handle, ling.data_ptr(), lens.data_ptr(), spk.data_ptr(), style.data_ptr(),
                                        content.data_ptr(), B, T, int(invariant), dur.data_ptr(), pitch.data_ptr(),
                                        energy.data_ptr(), lens32_ptr, mel_lens_ptr, ws1.data_ptr(), n1, st))
        else:
            _abi.check(lib.ev_am_phase1_prosody(self.handle, ling.data_ptr(), lens.data_ptr(), spk.data_ptr(), style.data_ptr(),
                                                content.data_ptr(), B, T, int(invariant), prosody.data_ptr(), dur.data_ptr(),
                                                pitch.data_ptr(), energy.data_ptr(), lens32_ptr, mel_lens_ptr, ws1.data_ptr(), n1,
                                                st))
        # the path's single host sync: the output length is data dependent (alignment.py:194-195).  Asynchronous copy into pinned
        # memory + a polled event instead of a blocking .cpu(): a blocking wait of a few milliseconds puts the thread to sleep, and its
        # wake-up latency (measured: 5-15 ms now and then on a busy host) would sit in the middle of the forward with the GPU idle.
        mel_lens_host = self._read_back(meta[B:])
        status = int(mel_lens_host[B + 1])
        if status:      # what nn.Embedding / the mask construction raise in the reference (checked on the device, read with the lengths)
            if status & 1:
                raise IndexError("inputs_ling holds token ids outside [0, %d)" % int(self.cfg.n_vocab))
            if status & 2:
                raise IndexError("inputs_speaker holds ids outside [0, %d)" % int(self.cfg.n_speaker))
            if status & 4:
                raise RuntimeError("input_lengths must lie in [1, %d] (the padded width of inputs_ling)" % T)
            if status & 16:
                raise ValueError("durations hold a negative value, or an utterance would have more frames than the vocoder can "
                                 "index (frames * %d must stay below 2^31); mel lengths %s"
                                 % (self.total_up, mel_lens_host[:B].tolist()))
            # the reference's decoder fails on a zero-length input (Conv1d raises); nothing of phase 2 has been enqueued
            raise RuntimeError("duration_scale leaves an utterance with no frames (mel lengths %s); use a larger duration_scale"
                               % mel_lens_host[:B].tolist())
        F = int(mel_lens_host[B])
        joined = {}
        need2 = lib.ev_phase2_workspace_bytes(self.handle, B, F)
        if group is not None:
            frames = group_frames(group, mel_lens_host[:B].numpy())
            if int(frames.max()) * self.total_up >= 2 ** 31:
                raise ValueError("a joined output would have more frames than the vocoder can index (frames * %d must stay below "
                                 "2^31); group lengths %s" % (self.total_up, frames.tolist()))
            lens_host = torch.from_numpy(frames.astype(np.int32))
            G, Fg = len(frames), int(frames.max())
            # The vocoder's kernels read their lengths before they wait for the kernel ahead of them (include/emotivoice_b200.h,
            # ev_vocoder), so the joined pass cannot take ev_join_mel's freshly written group_lens: it takes this upload, enqueued
            # before phase 2 and so complete before the vocoder's first kernel starts.
            joined = dict(group=group_dev, G=G, Fg=Fg, lens_host=lens_host, voc_lens=upload(lens_host))
            need2 = max(need2, lib.ev_phase2_workspace_bytes(self.handle, G, Fg))
        self.ensure_pe(F)
        ws2 = self._ws("p2", need2)
        n2 = ws2.numel()
        mel = torch.empty((B, F, int(self.cfg.n_mels)), dtype=torch.float32, device=dev)
        _abi.check(lib.ev_am_phase2(self.handle, ws1.data_ptr(), lens32_ptr, mel_lens_ptr, B, T, F, int(invariant),
                                    mel.data_ptr(), ws2.data_ptr(), n2, st))
        return dict(mel=mel, dur=dur, pitch=pitch, energy=energy, meta=meta, mel_lens=meta[B:2 * B],
                    mel_lens_host=mel_lens_host[:B], F=F, ws2=ws2, n2=n2, joined=joined)

    def vocode(self, mel, time_major, mel_lens_ptr, ws=None, n=0):
        lib, dev = self.lib, self.device
        if time_major:
            B, F, _ = mel.shape
        else:
            B, _, F = mel.shape
        if ws is None:
            ws = self._ws("p2", lib.ev_phase2_workspace_bytes(self.handle, B, F))
            n = ws.numel()
        wav = torch.empty((B, 1, F * self.total_up), dtype=torch.float32, device=dev)
        _abi.check(lib.ev_vocoder(self.handle, mel.data_ptr(), int(bool(time_major)), mel_lens_ptr, B, F,
                                  wav.data_ptr(), ws.data_ptr(), n, self._stream()))
        return wav

    def join_mel(self, mel, mel_lens, group, G, Fg):
        """ev_join_mel: (B,F,n_mels) mel + device (B,) frame counts and group ids -> joined (G,Fg,n_mels) mel, (G,) int32 lengths."""
        B, F, C = mel.shape
        joined = torch.empty((G, Fg, C), dtype=torch.float32, device=self.device)
        lens = torch.empty((G,), dtype=torch.int32, device=self.device)
        _abi.check(self.lib.ev_join_mel(mel.data_ptr(), mel_lens.data_ptr(), group.data_ptr(), B, F, C, G, Fg, joined.data_ptr(),
                                        lens.data_ptr(), self._stream()))
        return joined, lens


class _EngineOwner(nn.Module):
    """Lazy (re)packing of the parameter tree into an engine on the parameters' device."""

    def __init__(self):
        super().__init__()
        self._ev_engine = None
        self._ev_dirty = True
        self._ev_lock = threading.Lock()
        self._ev_precision = "fp32"
        self.register_load_state_dict_post_hook(_dirty_post_hook)

    @property
    def precision(self):
        """"fp32" (default): fp32-accurate 3xTF32 on the tensor cores (~1e-6 relative error).
        "tf32": decoder + vocoder with one tf32 MMA per K step (what the reference's eager PyTorch does for
        convolutions on a GPU); the duration-critical prefix stays fp32-accurate, so durations are
        identical in all modes.  "fp32_ffma": plain fp32 FFMA kernels, no tensor cores."""
        return self._ev_precision

    @precision.setter
    def precision(self, value):
        if value not in _abi.PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(_abi.PRECISIONS))
        self._ev_precision = value
        if self._ev_engine is not None:
            self._ev_engine.set_precision(value)
        for m in self.children():            # JETSGenerator.precision also governs .am / .generator used stand-alone
            if isinstance(m, _EngineOwner):
                m.precision = value

    def _mark_dirty(self):
        self._ev_dirty = True

    def _apply(self, fn, *a, **k):          # .to() / .cuda() / .float() ...
        r = super()._apply(fn, *a, **k)
        self._ev_dirty = True
        return r

    def refresh_weights(self):
        """Call after modifying parameters in place (load_state_dict / .to() do it for you)."""
        self._ev_dirty = True

    def _pack(self):
        raise NotImplementedError

    def attach_packed(self, blob, index_meta):
        """Adopt a packed weight blob produced elsewhere (rank 0 of a multi-GPU run) instead of packing this module's own
        parameters: ``blob`` is already on the module's device.  The caller guarantees it corresponds to the parameters."""
        dev = next(self.parameters()).device
        with self._ev_lock:
            self._ev_engine = _Engine(self.config, None, dev, self._ev_precision, blob=blob, index_meta=index_meta)
            self._ev_dirty = False
        return self._ev_engine

    def _engine(self):
        eng = self._ev_engine
        dev = next(self.parameters()).device
        if eng is not None and not self._ev_dirty and eng.device == dev:
            return eng
        with self._ev_lock:
            if self._ev_engine is None or self._ev_dirty or self._ev_engine.device != dev:
                self._ev_engine = _Engine(self.config, packing.add_tc_weights(self._pack()), dev, self._ev_precision)
                self._ev_dirty = False
            return self._ev_engine


def _prep(t, dtype, device):
    if t.device != device:
        raise RuntimeError("input tensor on %s but the module is on %s" % (t.device, device))
    if t.dtype != dtype:
        t = t.to(dtype)
    return t if t.is_contiguous() else t.contiguous()


def _seeded_init(conf):
    seed = int(torch.randint(0, 2 ** 31 - 1, ()).item())
    return synth.make_state_dict(conf, seed=seed)


class Generator(_EngineOwner):
    """HiFi-GAN generator (hifigan/models.py:90-140).  ``Generator(h)`` takes the ``model``
    node of the config, like the reference.  forward: (B, 80, F) -> (B, 1, 256 F)."""

    def __init__(self, h, _init=None):
        super().__init__()
        self.h = h
        self.num_kernels = len(h.resblock_kernel_sizes)
        self.num_upsamples = len(h.upsample_rates)
        self.upsample_factor = int(np.prod(h.upsample_rates))
        if str(h.resblock) != "1":
            raise NotImplementedError("only resblock '1' (config.yaml:87)")
        from .config import AttrDict
        self.config = AttrDict(model=h, n_mels=int(h.initial_channel), segment_size=32, n_vocab=1, n_speaker=1)
        if _init is None:
            full = AttrDict(model=h, n_mels=int(h.initial_channel), n_vocab=2, n_speaker=2)
            _init = {k[len("generator."):]: v for k, v in _seeded_init(full).items() if k.startswith("generator.")}
        for k, v in _init.items():
            _register(self, k, v.clone())
        self._register_load_state_dict_pre_hook(_legacy_weight_norm_hook, with_module=True)

    def _pack(self):
        return packing.pack_vocoder({"generator." + k: v for k, v in self.state_dict().items()}, self.h)

    @torch.no_grad()
    def forward(self, x):
        eng = self._engine()
        x = _prep(x, torch.float32, eng.device)
        with eng.call_lock:
            return eng.vocode(x, time_major=False, mel_lens_ptr=None)

    def remove_weight_norm(self):
        """hifigan/models.py:133-140 (broken on torch >= 2.1 in the reference, SURVEY.md s4-8):
        replaces every (g, v) pair by the folded ``weight``."""
        print('Removing weight norm...')
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        for mod, _, _ in synth.vocoder_conv_shapes(self.h):
            if mod + ".parametrizations.weight.original0" not in sd:
                continue
            w = packing.fold_weight_norm(sd, mod)
            holder = self
            for p in mod.split("."):
                holder = holder._modules[p]
            del holder._modules["parametrizations"]
            holder.register_parameter("weight", nn.Parameter(w.to(next(self.parameters()).device), requires_grad=False))
        self._mark_dirty()


class PromptTTS(_EngineOwner):
    """Acoustic model (model_open_source.py:14-163), inference branch only."""

    def __init__(self, config, _init=None):
        super().__init__()
        self.config = config
        if _init is None:
            _init = {k[len("am."):]: v for k, v in _seeded_init(config).items() if k.startswith("am.")}
        for k, v in _init.items():
            _register(self, k, v.clone())
        self.compat_padded_batch = False

    def _pack(self):
        sd = {"am." + k: v for k, v in self.state_dict().items()}
        packed = packing.pack_state_dict_am(sd, self.config)
        return packed

    @torch.no_grad()
    def forward(self, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding,
                mel_targets=None, output_lengths=None, pitch_targets=None, energy_targets=None, alpha=1.0,
                duration_scale=None, pitch_shift=None, energy_scale=None, durations=None, pitch=None, energy=None):
        """``duration_scale`` / ``pitch_shift`` / ``energy_scale`` and ``durations`` / ``pitch`` / ``energy``: prosody
        controls, see ``JETSGenerator.forward``."""
        if mel_targets is not None:
            raise NotImplementedError("training-mode forward (teacher forcing) is out of scope for this engine")
        prosody, given = controls_for(self, inputs_ling, duration_scale, pitch_shift, energy_scale, durations, pitch, energy)
        eng = self._engine()
        with eng.call_lock:
            return _am_forward(eng, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding,
                               inputs_content_embedding, not self.compat_padded_batch, prosody, given)[0]


def _am_forward(eng, inputs_ling, input_lengths, inputs_speaker, style, content, invariant, prosody=None, given=None, group=None):
    dev = eng.device
    ling = _prep(inputs_ling, torch.int64, dev)
    lens = _prep(input_lengths, torch.int64, dev)
    spk = _prep(inputs_speaker, torch.int64, dev)
    style = _prep(style, torch.float32, dev)
    content = _prep(content, torch.float32, dev)
    if ling.dim() != 2 or lens.dim() != 1 or lens.shape[0] != ling.shape[0] or spk.numel() != ling.shape[0]:
        raise RuntimeError("shape mismatch: inputs_ling %s, input_lengths %s, inputs_speaker %s"
                           % (tuple(ling.shape), tuple(lens.shape), tuple(spk.shape)))
    want = (ling.shape[0], int(eng.cfg.bert_dim))
    if tuple(style.shape) != want or tuple(content.shape) != want:
        raise RuntimeError("inputs_style_embedding %s / inputs_content_embedding %s must both be %s"
                           % (tuple(style.shape), tuple(content.shape), want))
    r = eng.acoustic(ling, lens, spk, style, content, invariant, prosody, given, group)
    out = {
        "mel_targets": None,
        "dec_outputs": r["mel"],
        "postnet_outputs": None,
        "pitch_predictions": r["pitch"].squeeze(),     # model_open_source.py:153
        "pitch_targets": None,
        "energy_predictions": r["energy"].squeeze(),   # :155
        "energy_targets": None,
        "log_duration_predictions": r["dur"],          # linear-domain integer frames despite the name (:157)
        "duration_targets": None,
        "input_lengths": input_lengths,
        "output_lengths": None,
        "log_p_attn": None,
        "bin_loss": None,
        "mel_lengths": r["mel_lens"],                  # extension: per-item frame counts (B,) int32
        "mel_lengths_host": r["mel_lens_host"],        # extension: the same on the host (read at the path's one sync)
    }
    return out, r


class JETSGenerator(_EngineOwner):
    """Joint acoustic model + vocoder (jets.py:26-71).

    ``compat_padded_batch`` (default False): with B > 1 the reference's padded forward leaks
    padding into the shorter items (decoder runs unmasked, convolutions run across pad frames;
    SURVEY.md s4 item 4).  By default every item of a batch is computed exactly like the
    reference's B=1 call for that item (what every reference caller runs); set the attribute
    to True to reproduce the literal padded-batch forward instead.  For B=1 both agree.

    Prosody controls (keyword arguments of ``forward``; each None, one float for every item, a length-B sequence / CPU
    tensor with one value per item, or a (B,T) nested sequence / CPU tensor with one value per phoneme, T =
    ``inputs_ling.shape[1]``):

    * ``duration_scale`` (1.0): multiplies the predicted durations before the length regulator -- the ``alpha`` of
      the reference's GaussianUpsampling (alignment.py:180-183).  Above 1 is slower speech; a server's ``speed``
      is ``duration_scale = 1 / speed``.
    * ``pitch_shift`` (0.0): semitones; the predicted pitch enters ``pitch_embed`` as the normalised pitch of
      2^(s/12) * f0, with the statistics of ``config.pitch_stats`` (default 225.089, 53.78).
    * ``energy_scale`` (1.0): multiplies frame energy the same way (``config.energy_stats``, default 30.610, 21.78).

    A per-phoneme value acts exactly where the per-item one acts, on its own token: token t's duration is
    fl32(fl32(d_t) * a_t), its pitch enters ``pitch_embed`` as p_t * r_t + shift_t.  Entries at t >= input_lengths[b]
    are ignored.  A per-phoneme ``duration_scale`` must lie in [1/16, 16] (a row holding one value throughout may hold
    any scale, as a per-item value may).  A table whose rows are constant gives
    bitwise the per-item result (under ``compat_padded_batch`` a per-phoneme table leaves the pad positions
    unshifted, where a per-item value shifts them too).

    Caller-given values (keyword arguments ``durations`` (integer frames), ``pitch``, ``energy`` (the predictors'
    normalised units)): each (B,T), or (T,) when B == 1, on the CPU or on the module's device.  They replace the
    predictions where those are used -- the durations in the length regulator, the tracks in ``pitch_embed`` /
    ``energy_embed`` -- and the controls above apply on top.  Values at t >= input_lengths[b] are ignored.  So the
    returned ``log_duration_predictions``, ``pitch_predictions`` and ``energy_predictions`` can be edited and passed
    back.  The all-zero guard of the length regulator applies to caller durations too.  Device durations are checked
    on the device: a negative one, or an utterance with more frames than the vocoder can index, raises ValueError
    before anything of the decoder is enqueued.

    The returned predictions stay the model's raw ones; ``mel_lengths`` counts the frames actually used.  Neutral
    values give bitwise the uncontrolled output.  Wrong shapes, dtypes or values raise ValueError before anything is
    enqueued.  ``alpha=`` is accepted and ignored, as in the reference's inference branch.  An utterance scaled to
    zero frames raises RuntimeError (the reference's decoder raises too).

    Long text (keyword argument ``join``): one group id per batch item, a sequence or CPU tensor of B integers, 0 first and
    each next one equal to the previous one or one more.  Consecutive items with one id are the segments of one output, in
    order (``frontdoor.split_phonemes`` cuts a long phoneme line into such segments).  The acoustic model runs over the B items
    exactly as without ``join``, with every control above; ``dec_outputs``, the predictions and ``mel_lengths`` stay per item.
    The vocoder then runs once per group over the items' valid mel rows concatenated, so its receptive field spans each seam
    and a group comes out as one continuous waveform: ``wav_predictions`` is (G, 1, hop * Fg), Fg the longest group's frames,
    and the result also holds ``joined_mel`` (G, Fg, n_mels, zeros past a group's length), ``joined_lengths`` ((G,) int32 on
    the device) and ``joined_lengths_host`` (the same on the host).  A group's waveform is bitwise what it gives in a forward
    of its own.  A malformed ``join``, or ``join`` with ``compat_padded_batch``, raises ValueError before anything is
    enqueued; a group too long for the vocoder's sample index raises ValueError before the decoder is enqueued.
    """

    def __init__(self, config):
        super().__init__()
        self.upsample_factor = int(np.prod(config.model.upsample_rates))
        self.segment_size = config.segment_size
        init = _seeded_init(config)
        self.am = PromptTTS(config, _init={k[3:]: v for k, v in init.items() if k.startswith("am.")})
        self.generator = Generator(config.model, _init={k[10:]: v for k, v in init.items() if k.startswith("generator.")})
        self.config = config
        self.compat_padded_batch = False
        self._register_load_state_dict_pre_hook(_legacy_weight_norm_hook, with_module=True)

    def _pack(self):
        return packing.pack_state_dict(self.state_dict(), self.config)

    @torch.no_grad()
    def forward(self, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding,
                mel_targets=None, output_lengths=None, pitch_targets=None, energy_targets=None, alpha=1.0,
                cut_flag=True, duration_scale=None, pitch_shift=None, energy_scale=None, durations=None, pitch=None, energy=None,
                join=None):
        if mel_targets is not None:
            raise NotImplementedError("training-mode forward (teacher forcing / random segments) is out of scope")
        prosody, given = controls_for(self, inputs_ling, duration_scale, pitch_shift, energy_scale, durations, pitch, energy)
        group = join_groups(join, int(inputs_ling.shape[0]))
        if group is not None and self.compat_padded_batch:
            raise ValueError("join needs per-item lengths: the literal padded forward (compat_padded_batch = True) has none")
        eng = self._engine()
        invariant = not self.compat_padded_batch
        with eng.call_lock:
            return self._forward_locked(eng, invariant, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding,
                                        inputs_content_embedding, prosody, given, group)

    def reserve(self, batch=1, phonemes=256, frames=2048):
        """Serving set-up: pre-size the engine's workspace arena (current CUDA stream) for requests up to this shape, so that no
        forward allocates device memory afterwards.  Without it the arena simply grows when a larger request arrives (one allocation
        stall per new maximum).  For joined traffic (``forward(join=...)``), ``frames`` counts a joined output's frames: the
        longest group's, not the longest segment's."""
        self._engine().reserve(batch, phonemes, frames)

    def _forward_locked(self, eng, invariant, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding, inputs_content_embedding,
                        prosody=None, given=None, group=None):
        outputs, r = _am_forward(eng, inputs_ling, input_lengths, inputs_speaker, inputs_style_embedding,
                                 inputs_content_embedding, invariant, prosody, given, group)
        B = r["mel"].shape[0]
        mel_lens_ptr = (r["meta"].data_ptr() + 4 * B) if invariant else None
        j = r["joined"]
        if j:
            # long text: the items' valid rows joined per group, then one vocoder pass over the G groups
            mel, lens = eng.join_mel(r["mel"], r["mel_lens"], j["group"], j["G"], j["Fg"])
            wav = eng.vocode(mel, time_major=True, mel_lens_ptr=j["voc_lens"].data_ptr(), ws=r["ws2"], n=r["n2"])
            outputs.update(joined_mel=mel, joined_lengths=lens, joined_lengths_host=j["lens_host"])
        else:
            # jets.py:62-66: z = dec_outputs.transpose(1, 2); wav = generator(z).  dec_outputs is already the
            # vocoder's time-major input layout: no transpose, no copy.
            wav = eng.vocode(r["mel"], time_major=True, mel_lens_ptr=mel_lens_ptr, ws=r["ws2"], n=r["n2"])
        outputs["wav_predictions"] = wav
        outputs["z_start_idxs"] = None
        outputs["segment_size"] = self.segment_size
        return outputs

    @torch.no_grad()
    def to_pcm16(self, wav):
        """The callers' ``wav * 32768 -> int16`` (inference_am_vocoder_joint.py:130-131) on the GPU: truncation toward zero
        like ``astype``.  Deviation: samples outside the int16 range SATURATE to [-32768, 32767] (tanh can round to exactly
        1.0 -> 32768) where numpy's cast wraps around; for |wav| < 1 the two agree bit for bit."""
        eng = self._engine()
        wav = _prep(wav, torch.float32, eng.device)
        pcm = torch.empty(wav.shape, dtype=torch.int16, device=eng.device)
        _abi.check(eng.lib.ev_wav_to_pcm16(wav.data_ptr(), pcm.data_ptr(), wav.numel(), eng._stream()))
        return pcm

    def _outputs(self, out, items, hop):
        """The outputs of a forward as ``format_audio`` takes them -> (wav, n_in, items, engine), or ValueError."""
        wav = out["wav_predictions"]
        if not (isinstance(wav, torch.Tensor) and wav.dim() == 3 and wav.dtype == torch.float32 and wav.is_contiguous()):
            raise ValueError("out['wav_predictions'] must be a contiguous (B, 1, L) float32 tensor")
        B, width = int(wav.shape[0]), int(wav.shape[-1])
        hop = self.upsample_factor if hop is None else int(hop)
        lens = out.get("joined_lengths_host")
        if lens is None:
            lens = out.get("mel_lengths_host")
        n_in = [width] * B if lens is None else [min(width, int(v) * hop) for v in lens.tolist()]
        if len(n_in) != B:
            raise ValueError("out holds %d lengths for %d waveforms" % (len(n_in), B))
        if items is None:
            items = list(range(B))
        else:
            items = [int(i) for i in items]
            if not items or any(i < 0 or i >= B for i in items):
                raise ValueError("items must be a non-empty list of output indices in [0, %d), got %s" % (B, items))
        if len(items) > 65535:
            raise ValueError("format_audio takes at most 65535 outputs per call, got %d" % len(items))
        eng = self._engine()
        if wav.device != eng.device:
            raise ValueError("out['wav_predictions'] is on %s but the module is on %s" % (wav.device, eng.device))
        return wav, n_in, items, eng

    @torch.no_grad()
    def measure_loudness(self, out, items=None, hop=None):
        """Integrated loudness (ITU-R BS.1770-4, LUFS) and sample peak of each output of a forward, on the GPU, at the model's
        rate.  ``out`` / ``items`` / ``hop``: the outputs ``format_audio`` would encode (a joined forward's groups are measured
        as one waveform each).  Returns (lufs, peak): device float32 tensors of len(items); lufs is -inf for an output shorter
        than 400 ms or with no 400 ms block above the gates (silence).  No sync."""
        wav, n_in, items, eng = self._outputs(out, items, hop)
        with eng.call_lock:
            return eng.output.measure(wav, n_in, items, int(getattr(self.config, "sr", 16000)))

    @torch.no_grad()
    def meter(self, out, sample_rate=None, items=None, hop=None, loudness=None, true_peak=None, watermark=None, series=False):
        """The loudness meter (EBU R128; ``emotivoice_b200.loudness`` holds the definitions) of exactly what
        ``format_audio(out, sample_rate, "float32", items, hop, loudness, true_peak, watermark)`` delivers: the chain's float32
        stage runs as it would there, then ``ev_meter`` reads its packed outputs in place, at the output rate.  Lets a server
        check the integrated loudness, true peak, maximum momentary and short-term loudness and loudness range of its
        responses.  The output rate must also be a multiple of 10 Hz (100 ms sub-blocks).  ``series``: also return the
        momentary and short-term series.

        Returns a ``loudness.Meter`` of device tensors, one value per listed output.  No sync; invalid arguments raise
        ValueError before anything is enqueued."""
        sr = int(getattr(self.config, "sr", 16000))
        fmt = audio.output_format(sample_rate, "float32", loudness, true_peak, sr, watermark=watermark)
        check_meter_rate(fmt.rate)
        if not isinstance(series, (bool, np.bool_)):
            raise ValueError("series must be True or False, got %r" % (series,))
        wav, n_in, items, eng = self._outputs(out, items, hop)
        with eng.call_lock:
            packed, offs = eng.output.format(wav, n_in, items, fmt, sr)
            return eng.output.meter(packed, offs, fmt.rate, bool(series))

    @torch.no_grad()
    def format_audio(self, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None,
                     watermark=None):
        """The output of a forward in a client's format, on the GPU: each output's valid samples, resampled to ``sample_rate``
        (None: the model's rate, ``config.sr``, 16000) and encoded, packed back to back.

        ``out`` is the dict ``forward`` returned: output b is ``wav_predictions[b]`` trimmed to ``joined_lengths_host[b] * hop``
        for a joined forward, else ``mel_lengths_host[b] * hop`` (hop: ``upsample_factor`` unless given), else its full width.
        ``items``: the outputs to format, in order (default: all).  ``encoding``: "float32", "pcm16" (trunc(y * 32768),
        saturated, as ``to_pcm16``), "mulaw" or "alaw" (one byte of G.711 of that int16 value).  Resampling is
        ``scipy.signal.resample_poly(x, up, down)`` with its default filter, up / down the reduced ratio of the two rates, each
        at most 1024 (see ``audio.plan``); fp32 arithmetic, one chain per sample in tap order, so an output does not depend on
        the others.  At the model's rate "float32" is the trimmed waveform itself and "pcm16" ``to_pcm16`` of it, bit for bit.

        ``loudness`` (a target in LUFS, in [-70, 0], or None): each output is first measured as ``measure_loudness`` does and
        scaled by g = min(10^((loudness - L) / 20), 10^(-1/20) / peak) before it is resampled and encoded (a -1 dBFS sample-peak
        ceiling; g = 1 where L = -inf).  g is computed in fp64 and applied in fp32 as fp32(y * g), y the resampled sample; the
        gain is the same at every output rate, since resampling is linear.  None: no measurement, and the output is exactly
        as without the argument.

        ``true_peak`` (a ceiling in dBTP, in [-20, 0], or None): a look-ahead limiter holds each output at or below the ceiling
        in true peak (``ev_limit``, run at the model's rate before resampling).  Its pre-gain is 10^((loudness - L) / 20) with no
        sample-peak cap (1 without ``loudness`` or where L = -inf).  With ``loudness``, two passes: the limited output is measured
        again (L1) and the original samples are limited once more under the pre-gain times 10^((loudness - L1) / 20), so the
        target is reached where limiting took loudness away.  The detector oversamples to 192 kHz (12x at 16 kHz) and, for a
        rate below the model's, also low-passes as the resampler does; look-ahead 5 ms, linear release 60 dB/s.  The limited
        waveform is then resampled and encoded with no further gain.  None: the limiter does not run, and the output is exactly
        as without the argument.

        ``watermark`` (an integer key in [1, 2^63 - 1], or None): before anything else, each output gets a keyed mark that
        ``emotivoice_b200.watermark.detect`` finds again (``ev_watermark_embed``, at the model's rate; see ``audio`` for its
        constants): in each 1024-sample MCLT frame, bins of about 300-3400 Hz are changed by a keyed +-1 pattern 20 dB under
        their own magnitude.  Loudness, the limiter, resampling and encoding then process the marked output, so their targets
        hold for what is delivered.  Needs an output rate of at least 8000 Hz.  None: the output is exactly as without the
        argument.

        ``encoding="flac"``: each output becomes a complete .flac file image (RFC 9639: mono, 16 bits, 4096-sample blocks) of
        exactly the samples "pcm16" gives, encoded on the GPU by ev_flac_encode; decoding it returns that PCM16 bit for bit.
        The images' sizes exist only after encoding, so this encoding makes ONE device->host read of the len(items) + 1
        offsets (a sync); every other encoding is sync-free.

        Returns (packed 1-D device tensor: float32, int16 or uint8; (len(items) + 1,) int64 numpy offsets: output k is
        ``packed[offs[k]:offs[k + 1]]``).  No sync except for "flac": the lengths are the host copies the forward read.
        Invalid arguments raise ValueError before anything is enqueued."""
        sr = int(getattr(self.config, "sr", 16000))
        fmt = audio.output_format(sample_rate, encoding, loudness, true_peak, sr, watermark=watermark)
        wav, n_in, items, eng = self._outputs(out, items, hop)
        if encoding == audio.FLAC and any(n_in[b] < 1 for b in items):
            raise ValueError("an output with no samples cannot be a FLAC stream (valid samples %s)" % [n_in[b] for b in items])
        with eng.call_lock:
            return eng.output.format(wav, n_in, items, fmt, sr)
