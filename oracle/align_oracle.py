"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the training-mode alignment helpers (SURVEY.md s8f rank 4):
monotonic alignment search, its duration / bin-loss post-processing and the per-token averaging of frame-level targets
(models/prompt_tts_modified/modules/alignment.py:90-177).  The reference runs them per sample in numba on the CPU, between
GPU stages of the training step.  Pinned against the reference's own numba functions by oracle/make_golden_align.py.

Arithmetic that decides the (integer) path, restated exactly:
  * log_p_attn arrives as float32; Q is float64 (np.full default); row 0 is the float32 running sum of log_prob[0, :j+1]
    (numba sums a float32 slice sequentially in float32) widened to float64; every other cell is a float64 max + float32 add;
  * cells with i > j keep -inf; the backtrack prefers the SMALLER token index on ties (`Q[i_a, j] >= Q[i_b, j]`).
The per-token averages are restated with the reference's arithmetic too (a sequential float32 sum over numpy slice
semantics), so they equal its output bit for bit; ``average_by_duration64`` and ``align_logp64`` are the float64 references
the GPU tests bound the kernels against.
"""
import numpy as np


def monotonic_alignment_search(log_p_attn, return_q=False):
    """(T_mel, T_inp) float32 -> (T_mel,) int64 token index per frame (alignment.py:90-121) [, the score table Q (T_inp, T_mel)]."""
    lp = np.ascontiguousarray(log_p_attn, dtype=np.float32).T          # (T_inp, T_mel)
    T_inp, T_mel = lp.shape
    Q = np.full((T_inp, T_mel), -np.inf, dtype=np.float64)
    Q[0] = np.cumsum(lp[0], dtype=np.float32).astype(np.float64)       # sequential float32 prefix sums
    for j in range(1, T_mel):
        hi = min(j + 1, T_inp)
        if hi > 1:
            Q[1:hi, j] = np.maximum(Q[0:hi - 1, j - 1], Q[1:hi, j - 1]) + lp[1:hi, j].astype(np.float64)
    A = np.full((T_mel,), T_inp - 1, dtype=np.int64)
    for j in range(T_mel - 2, -1, -1):
        i_b = A[j + 1]
        i_a = i_b - 1
        if i_b == 0:
            A[j] = 0
        elif Q[i_a, j] >= Q[i_b, j]:
            A[j] = i_a
        else:
            A[j] = i_b
    return (A, Q) if return_q else A


def mix32(seed, n):
    """n pseudo-random uint32 from a splitmix64 counter: integer arithmetic only, so every host draws the same bits."""
    z = (np.arange(n, dtype=np.uint64) + np.uint64(1) + np.uint64(seed) * np.uint64(1 << 32)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return ((z ^ (z >> np.uint64(31))) >> np.uint64(32)).astype(np.int64)


MAS_KINDS = ("band", "ties", "ninf")


def band_log_p(text_lengths, feats_lengths, T_pad, F_pad, seed, kind="band"):
    """(B, F_pad, T_pad) float32 alignment scores shaped like a trained aligner's: a diagonal band from (0, 0) to each item's
    (feats_length, text_length) corner plus noise, every value an integer times a power of two (exact, no transcendentals).
    "band": 0.5 per token off the diagonal, noise up to 2, about 23 significant bits (float32 row sums round);
    "ties": 1 per token, noise 0..1 in steps of 0.5, so equal predecessor scores are frequent;
    "ninf": "band" with about one cell in 23 set to -inf, inside the item's rectangle too."""
    B = len(text_lengths)
    r = mix32(seed, B * F_pad * T_pad).reshape(B, F_pad, T_pad)
    i = np.arange(T_pad, dtype=np.int64)[None, :]
    j = np.arange(F_pad, dtype=np.int64)[:, None]
    out = np.empty((B, F_pad, T_pad), np.float32)
    for b in range(B):
        T, F = max(int(text_lengths[b]), 1), max(int(feats_lengths[b]), 1)
        dist = np.abs((2 * i + 1) * F - (2 * j + 1) * T)                     # 2 F |i + 1/2 - (j + 1/2) T / F|
        if kind == "ties":
            k = dist // (2 * F) * 2 + r[b] % 3
            out[b] = -k.astype(np.float32) * np.float32(0.5)
        else:
            k = dist * (1 << 14) // (2 * F) + r[b] % (1 << 16)              # < 2^24 for T_pad <= 1023: exact in float32
            out[b] = -k.astype(np.float32) * np.float32(2.0 ** -15)
            if kind == "ninf":
                out[b][(r[b] >> 16) % 23 == 0] = -np.inf
    return out


def viterbi_decode(log_p_attn, text_lengths, feats_lengths):
    """(B, T_mel, T_inp) float32 -> durations (B, T_inp) float32, bin_loss scalar (alignment.py:124-142)."""
    B, _, T_text = log_p_attn.shape
    ds = np.zeros((B, T_text), np.float32)
    bin_loss = 0.0
    for b in range(B):
        cur = log_p_attn[b, :feats_lengths[b], :text_lengths[b]]
        path = monotonic_alignment_search(cur)
        cnt = np.bincount(path)
        ds[b, :len(cnt)] = cnt
        bin_loss = bin_loss - np.float32(cur[np.arange(feats_lengths[b]), path].astype(np.float32).mean(dtype=np.float32))
    return ds, np.float32(bin_loss / B)


def _token_slices(ds, xs, text_lengths, feats_lengths):
    """Yields (b, n, x[start:end]) for every token the reference averages: durations truncated to int32, start / end the
    exclusive / inclusive cumulative sums, the slice taken with numpy's semantics (a negative bound counts from the end of the
    length-feats_lengths[b] row, both then clip to it) exactly as the reference's numba loop takes it."""
    d = np.asarray(ds).astype(np.int32)
    for b in range(d.shape[0]):
        cs = [0] + list(np.cumsum(d[b, :int(text_lengths[b])]))
        x = np.asarray(xs[b, :int(feats_lengths[b])], np.float32)
        for n, (s, e) in enumerate(zip(cs[:-1], cs[1:])):
            yield b, n, x[int(s):int(e)]


def average_by_duration(ds, xs, text_lengths, feats_lengths):
    """Per-token mean of a frame-level track over the token's frames; 0 for empty slices (alignment.py:145-177), with the
    reference's arithmetic: numba's float32 ``x[s:e].mean()`` is the sequential float32 sum, divided by n in float64, stored
    as float32.  Equal bit for bit to the reference's output (oracle/make_golden_align.py asserts it on every fixture)."""
    out = np.zeros(np.shape(ds), dtype=np.float32)
    for b, n, seg in _token_slices(ds, xs, text_lengths, feats_lengths):
        if len(seg):
            out[b, n] = np.float32(np.float64(np.cumsum(seg, dtype=np.float32)[-1]) / np.float64(len(seg)))
    return out


def average_by_duration64(ds, xs, text_lengths, feats_lengths):
    """The same slices' means in float64 (the float32 inputs widened, summed with fsum: correctly rounded); 0 for empty slices."""
    import math
    out = np.zeros(np.shape(ds), dtype=np.float64)
    for b, n, seg in _token_slices(ds, xs, text_lengths, feats_lengths):
        if len(seg):
            out[b, n] = math.fsum(seg.astype(np.float64).tolist()) / len(seg)
    return out


def align_logp64(text, feats, text_lens=None, prior=None):
    """The distance / masked log-softmax / prior stage of AlignmentModule.forward (alignment.py:41-54) in float64, as torch on
    any device.  text (B, T, A), feats (B, F, A); tokens t >= text_lens[b] are masked (None: no mask); prior (B, F, T) or None.
    Returns (log_p (B, F, T), |score| (B, F, T), |lse| (B, F, 1)): the magnitudes are the terms an error bound scales with."""
    import torch
    t = text.to(torch.float64)
    f = feats.to(torch.float64)
    B, T, _ = t.shape
    score = -torch.cdist(f, t, p=2.0, compute_mode="donot_use_mm_for_euclid_dist")       # direct differences: no |a|^2 + |b|^2 - 2ab
    if text_lens is not None:
        tl = text_lens.to(score.device).clamp(0, T)
        score = score.masked_fill(torch.arange(T, device=score.device)[None, None, :] >= tl[:, None, None], -np.inf)
    lse = torch.logsumexp(score, dim=-1, keepdim=True)
    lp = score - lse
    if prior is not None:
        lp = lp + prior.to(device=lp.device, dtype=torch.float64)
    return lp, score.abs(), lse.abs()


def alignment_module_forward(sd, text, feats, text_lengths, feats_lengths, x_masks=None, prefix="", prior_fn=None):
    """AlignmentModule.forward (alignment.py:33-56) as plain functional torch on the CPU.  ``sd``: the module's state dict
    (t_conv1.weight ...).  The prior comes from ``prior_fn(text_lengths, feats_lengths)`` (the product's host code builds it with
    the same scipy call as the reference; passing the reference's own here keeps this function a pure restatement)."""
    import torch
    import torch.nn.functional as F
    g = lambda n: sd[prefix + n]
    t = text.transpose(1, 2)
    t = F.relu(F.conv1d(t, g("t_conv1.weight"), g("t_conv1.bias"), padding=1))
    t = F.conv1d(t, g("t_conv2.weight"), g("t_conv2.bias")).transpose(1, 2)
    f = feats.transpose(1, 2)
    f = F.relu(F.conv1d(f, g("f_conv1.weight"), g("f_conv1.bias"), padding=1))
    f = F.relu(F.conv1d(f, g("f_conv2.weight"), g("f_conv2.bias"), padding=1))
    f = F.conv1d(f, g("f_conv3.weight"), g("f_conv3.bias")).transpose(1, 2)
    score = -torch.norm(f.unsqueeze(2) - t.unsqueeze(1), p=2, dim=3)
    if x_masks is not None:
        score = score.masked_fill(x_masks.unsqueeze(-2), -np.inf)
    lp = F.log_softmax(score, dim=-1)
    return lp + prior_fn(text_lengths, feats_lengths).to(lp.dtype) if prior_fn is not None else lp


def get_segments(x, start_idxs, segment_size):
    """models/hifigan/get_random_segments.py:19-27 in numpy: (B, C, T) -> (B, C, segment_size), zero padded."""
    B, C, T = x.shape
    out = np.zeros((B, C, segment_size), x.dtype)
    for b in range(B):
        s = int(start_idxs[b])
        seg = x[b, :, s:s + segment_size]
        out[b, :, :seg.shape[1]] = seg
    return out
