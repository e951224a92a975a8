"""Training-mode alignment helpers on the GPU (SURVEY.md s8f rank 4) with the reference's function names and signatures
(models/prompt_tts_modified/modules/alignment.py:124-177): ``viterbi_decode`` and ``average_by_duration``.

The reference copies ``log_p_attn`` to the host and runs a numba loop per sample in the middle of every training step
(model_open_source.py:114-118); here one kernel launch handles the batch and nothing leaves the device.  Paths and durations are
bit-exact with the reference (the kernel restates its float64 dynamic programme).  ``bin_loss`` and the averages are float32
roundings of float64 means: within 1 ulp of the exact mean.  The reference's averages are float32 running sums (numba), which
drift from the exact mean by a few ulp at the magnitudes of energy and pitch tracks; durations that sum past the track clip to
it, and negative durations slice the track the way numpy does, as in the reference.

Also here (the rest of SURVEY.md s8f rank 4): ``AlignmentModule`` (alignment.py:13-87: five convolutions on the tensor cores in
the fp32-accurate 3xTF32 mode, the L2-distance / masked log-softmax kernel, the beta-binomial prior built on the host exactly
like the reference builds it) and ``get_random_segments`` / ``get_segments`` (models/hifigan/get_random_segments.py, used by
jets.py:55-60).  Forward only: losses and autograd stay out of scope.
"""
import numpy as np
import torch
import torch.nn as nn

from . import _abi, packing


def _check(t, name):
    if t.device.type != "cuda":
        raise RuntimeError("%s must be a CUDA tensor: emotivoice_b200 has no CPU path" % name)


def viterbi_decode(log_p_attn, text_lengths, feats_lengths, return_path=False):
    """log_p_attn (B, T_feats, T_text) float32 -> (ds (B, T_text) float32, bin_loss 0-dim float32)  [+ path (B, T_feats) int32]."""
    _check(log_p_attn, "log_p_attn")
    lib = _abi.load()
    dev = log_p_attn.device
    lp = log_p_attn.detach().to(torch.float32).contiguous()
    B, F, T = lp.shape
    tl = text_lengths.to(device=dev, dtype=torch.int64).contiguous()
    fl = feats_lengths.to(device=dev, dtype=torch.int64).contiguous()
    path = torch.empty((B, F), dtype=torch.int32, device=dev)
    ds = torch.empty((B, T), dtype=torch.float32, device=dev)
    loss = torch.empty((B,), dtype=torch.float32, device=dev)
    ws = torch.empty((B * F * T,), dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_op_mas(lp.data_ptr(), tl.data_ptr(), fl.data_ptr(), B, F, T, path.data_ptr(), ds.data_ptr(), loss.data_ptr(),
                             ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream))
    bin_loss = loss.sum() / B                      # alignment.py:141: the per-item means, averaged over the batch
    return (ds, bin_loss, path) if return_path else (ds, bin_loss)


def average_by_duration(ds, xs, text_lengths, feats_lengths):
    """ds (B, T_text), xs (B, T_feats) -> (B, T_text) float32: mean of xs over each token's frames (0 for empty tokens)."""
    _check(ds, "ds")
    lib = _abi.load()
    dev = ds.device
    d = ds.detach().to(torch.float32).contiguous()
    x = xs.detach().to(device=dev, dtype=torch.float32).contiguous()
    B, T = d.shape
    F = x.shape[1]
    tl = text_lengths.to(device=dev, dtype=torch.int64).contiguous()
    fl = feats_lengths.to(device=dev, dtype=torch.int64).contiguous()
    out = torch.empty((B, T), dtype=torch.float32, device=dev)
    _abi.check(lib.ev_op_average_by_duration(d.data_ptr(), x.data_ptr(), tl.data_ptr(), fl.data_ptr(), B, F, T, out.data_ptr(),
                                             torch.cuda.current_stream(dev).cuda_stream))
    return out


class AlignmentModule(nn.Module):
    """alignment.py:13-56 with the reference's constructor, parameter names (``t_conv1.weight`` ...) and forward signature.
    ``text`` (B, T_text, adim), ``feats`` (B, T_feats, odim) -> ``log_p_attn`` (B, T_feats, T_text).  Forward only.
    ``x_masks`` must be a suffix mask (True from each item's text length on, as model_open_source.py builds it): only its count
    of unmasked tokens per item is used."""

    CONVS = (("t_conv1", 3), ("t_conv2", 1), ("f_conv1", 3), ("f_conv2", 3), ("f_conv3", 1))

    def __init__(self, adim, odim, cache_prior=True):
        super().__init__()
        self.adim, self.odim, self.cache_prior = int(adim), int(odim), cache_prior
        self._cache = {}
        for name, k in self.CONVS:
            cin = self.odim if name == "f_conv1" else self.adim
            holder = nn.Module()
            bound = 1.0 / np.sqrt(cin * k)
            holder.register_parameter("weight", nn.Parameter(torch.empty(self.adim, cin, k).uniform_(-bound, bound), requires_grad=False))
            holder.register_parameter("bias", nn.Parameter(torch.empty(self.adim).uniform_(-bound, bound), requires_grad=False))
            self.add_module(name, holder)
        self._packed = None

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._packed = None
        return r

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self._packed = None
        return r

    def _weights(self, dev):
        if self._packed is None or self._packed[0] != dev:
            w = {}
            for name, _ in self.CONVS:
                m = getattr(self, name)
                w[name] = (packing.to_tc_layout(packing._conv_w(m.weight.detach().float().cpu())).to(dev), m.bias.detach().float().to(dev).contiguous())
            self._packed = (dev, w)
        return self._packed[1]

    def _conv(self, lib, x, name, k, relu, st):
        w, b = self._weights(x.device)[name]
        B, L, cin = x.shape
        out = torch.empty((B, L, self.adim), dtype=torch.float32, device=x.device)
        _abi.check(lib.ev_op_conv1d_tc(x.data_ptr(), w.data_ptr(), 1, b.data_ptr(), 0, None, out.data_ptr(), B, L, cin, self.adim, k, 1, None, 1,
                                       _abi.ACT_NONE, 0.0, _abi.ACT_RELU if relu else _abi.ACT_NONE, _abi.ACC_STORE, 1.0, None, 0, st))
        return out

    @torch.no_grad()
    def forward(self, text, feats, text_lengths, feats_lengths, x_masks=None):
        _check(text, "text")
        lib = _abi.load()
        dev = text.device
        st = torch.cuda.current_stream(dev).cuda_stream
        text = text.detach().float().contiguous()
        feats = feats.detach().to(dev).float().contiguous()
        if self.odim % 8 or self.adim % 128:
            raise ValueError("AlignmentModule on the tensor cores needs odim % 8 == 0 and adim % 128 == 0")
        t = self._conv(lib, text, "t_conv1", 3, True, st)          # the module's layout is already time-major: no transposes
        t = self._conv(lib, t, "t_conv2", 1, False, st)
        f = self._conv(lib, feats, "f_conv1", 3, True, st)
        f = self._conv(lib, f, "f_conv2", 3, True, st)
        f = self._conv(lib, f, "f_conv3", 1, False, st)
        B, F, T = f.shape[0], f.shape[1], t.shape[1]
        tl = None
        if x_masks is not None:                                    # True = padded token (model_open_source.py:164-173): a suffix mask
            tl = (~x_masks.to(dev).bool()).sum(dim=-1).to(torch.int64).contiguous()
        prior = self._generate_prior(text_lengths, feats_lengths).to(device=dev, dtype=torch.float32)
        if prior.shape != (B, F, T):                               # the reference adds by broadcasting identical shapes
            raise RuntimeError("prior %s vs log_p_attn %s: text / feats are not padded to their maximum lengths" % (tuple(prior.shape), (B, F, T)))
        prior = prior.contiguous()
        out = torch.empty((B, F, T), dtype=torch.float32, device=dev)
        _abi.check(lib.ev_op_align_logp(t.data_ptr(), f.data_ptr(), None if tl is None else tl.data_ptr(), prior.data_ptr(), B, F, T, self.adim,
                                        out.data_ptr(), st))
        return out

    def _generate_prior(self, text_lengths, feats_lengths, w=1):
        """alignment.py:58-87: log beta-binomial pmf over tokens for every frame, cached per (T_feats, T_text)."""
        from scipy.stats import betabinom
        B = len(text_lengths)
        T_text, T_feats = int(max(int(v) for v in text_lengths)), int(max(int(v) for v in feats_lengths))
        bb_prior = torch.full((B, T_feats, T_text), fill_value=-np.inf)
        for bidx in range(B):
            T, N = int(feats_lengths[bidx]), int(text_lengths[bidx])
            key = "%d,%d" % (T, N)
            prob = self._cache.get(key) if self.cache_prior else None
            if prob is None:
                alpha = w * np.arange(1, T + 1, dtype=float)
                beta = w * np.array([T - t + 1 for t in alpha])
                prob = betabinom.logpmf(np.arange(N)[..., None], N, alpha, beta)       # (N, T)
                if self.cache_prior:
                    self._cache[key] = prob
            bb_prior[bidx, :T, :N] = torch.from_numpy(prob).transpose(0, 1)
        return bb_prior


def get_segments(x, start_idxs, segment_size):
    """models/hifigan/get_random_segments.py:19-27: x (B, C, T) -> (B, C, segment_size), zero padded past T."""
    _check(x, "x")
    lib = _abi.load()
    x = x.detach().float().contiguous()
    B, C, T = x.shape
    start = start_idxs.to(device=x.device, dtype=torch.int64).contiguous()
    out = torch.empty((B, C, int(segment_size)), dtype=torch.float32, device=x.device)
    _abi.check(lib.ev_op_get_segments(x.data_ptr(), start.data_ptr(), B, C, T, int(segment_size), out.data_ptr(),
                                      torch.cuda.current_stream(x.device).cuda_stream))
    return out


def get_random_segments(x, x_lengths, segment_size):
    """models/hifigan/get_random_segments.py:8-16 (jets.py:55-60): the start indices are drawn with the same torch calls as
    the reference (``torch.rand([b])`` on the default CPU generator), so a seeded run picks the same segments."""
    b = x.shape[0]
    max_start_idx = torch.clamp(x_lengths.to(x.device) - segment_size, min=0)
    start_idxs = (torch.rand([b]).to(x.device) * max_start_idx).to(dtype=torch.long)
    return get_segments(x, start_idxs, segment_size), start_idxs, segment_size
