"""fp64 references of the plain fp32 kernels between the acoustic model's GEMMs and of the style encoder's own kernels, the
per-element magnitudes they are judged by, the launch rules that pick their instantiations, and the operator cases of
tests/test_fp32_kernels_gpu.py.

Like tests/am_ref.py, every reference returns, next to each output element y64, a magnitude m such that a kernel whose fp32
operations each add a relative error of a few ulps is off by at most ~u * m there, whatever the cancellation.  Every kernel here
is fp32 FFMA code, so every element is held to the fp32-accurate class, |y - y64| <= TAU * m with TAU = 2^-14 (voc_ref.TAU[1]),
and the whole result to REL_MAX = voc_ref.REL_MAX[1] of max|y64|.  The longest fp32 chain is cond_gemv's: each thread adds
1920 / 256 = 8 products, a lane of the reduce adds 32 partials and the shuffles 3 more, ~43 ulps = 2^-18.5 m; the bound leaves
room for 16 times that and for the transcendental functions' few ulps.  The magnitudes:

* GEMV (cond_gemv, row_gemv, rowdot):  y = act(bias + sum_k w_k x_k),  m = |bias| + sum_k |w_k| |x_k|.  act is none or tanh,
  whose Lipschitz constant is 1, so the pre-activation bound holds after it.
* LayerNorm, eps 1e-12, biased variance, per row of C channels:  y = w x^ + b,  x^ = (x - mu) / sigma,  sigma = sqrt(var + eps),
      m = |w| (|x^| + (mean|x| / sigma)(1 + |x^|)) + |b|.
  |x^| carries the rounding of x - mu, of the product chain and of rstd's relative error.  The mean is a sum of C terms of size up
  to mean|x| C, so its error is ~u mean|x|.  It moves x - mu by that much, hence the term (mean|x| / sigma) in x^.  It also moves
  the variance, so rstd's relative error gets the same term, times |x^|.  The prologue's x is taken as the kernel writes it:
  fl32(e + fl32(alpha * pe)), bitwise equal to torch's fp32 `emb[id] + alpha * pe[t]`.
* var_embed_add (K taps, window [t - (K-1)/2, t + (K-1)/2] clipped to [0, tl)):
      y = x + (sum_j wp_j p'_j + bp) + (sum_j we_j e'_j + be),   m = |x| + |bp| + sum |wp||p'| + |be| + sum |we||e'|
  with p', e' the tracks after the fp32 prosody affine (the values the convolution reads, computed in fp32 like the kernel).
* Gaussian upsampling of frame f over the item's tokens t < tlen, like attention (am_ref.attn_ref):
      e_t = -fl32(0.1) (f - c_t)^2,   p = softmax(e),   o = sum_t p_t h_t (+ alpha pe[f]),
      m = sum_t p_t |h_t| + sum_t p_t |e_t| |h_t - o| (+ |alpha pe[f]|).
  An error of a few ulps of e_t (f - c_t, the square, the product, e_t - max) moves o by p_t u |e_t| (h_t - o): the score term.
* Durations (rowdot mode 1): s64 = b + sum x w, d = clamp(rint(exp(s64) - 1), 0).  The kernel's s lies within TAU m of s64 and
  its exp within a few ulps, so where [s64 - TAU m, s64 + TAU m], widened by 4 ulps of exp, straddles a rounding boundary
  ln(k + 1.5) both neighbours are accepted.  At random data that band holds a fraction of a percent of the rows.
"""
import math

import torch

import am_ref
import voc_ref

TAU, REL_MAX = voc_ref.TAU[1], voc_ref.REL_MAX[1]
EPS = 1e-12
TENTH32 = float(torch.tensor(0.1, dtype=torch.float32))     # the kernel's 0.1f
EXP_ULPS = 4 * 2.0 ** -23


def check(y, y64, m, rel_max=None):
    """-> dict(err_m, rel_max, ok): every element within TAU * m, the whole within REL_MAX of max|y64|."""
    return am_ref.check(y, y64, m, 1, rel_max)


# ---- references ------------------------------------------------------------------------------------------------------------
def gemv_ref(x, w, bias, tanh=False):
    """x (B, K), w (K, N), bias (N,) -> (y, m), each (B, N)."""
    xd, wd, bd = x.double(), w.double(), bias.double()
    y = xd @ wd + bd
    m = xd.abs() @ wd.abs() + bd.abs()
    return (torch.tanh(y) if tanh else y), m


def cond_input(spk, spk_emb, style, content):
    """The gathered conditioning vectors (B, H + 2 bert), fp32, speaker ids clamped like the kernel."""
    sid = spk.clamp(0, spk_emb.shape[0] - 1)
    return torch.cat([spk_emb[sid], style, content], 1)


def ln_ref(x, w, b):
    """LayerNorm over the last dim of x (rows, C) -> (y, m)."""
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    sig = (var + EPS).sqrt()
    xh = (xd - mu) / sig
    wd, bd = w.double(), b.double()
    m = wd.abs() * (xh.abs() + xd.abs().mean(-1, keepdim=True) / sig * (1 + xh.abs())) + bd.abs()
    return xh * wd + bd, m


def ln_check(y, x, w, b):
    """LayerNorm output y (rows, C) of input x: every element within TAU * m, and REL_MAX of max|y64| over the rows whose
    mean|x| is at most 4 sigma.  Where the mean is far above sigma the input's conditioning, not the kernel, sets the error
    relative to max|y64| (an fp32 mean of values near 100 is off by ~1e-5), and only the per-element bound can judge it."""
    y64, m = ln_ref(x, w, b)
    r = check(y, y64, m, rel_max=math.inf)
    xd = x.double()
    calm = xd.abs().mean(-1) <= 4 * (xd.var(-1, unbiased=False) + EPS).sqrt()
    r2 = check(y[calm], y64[calm], m[calm])
    return dict(err_m=r["err_m"], rel_max=r2["rel_max"], ok=r["ok"] and r2["ok"])


def ln_input(rows, C, g):
    """LayerNorm input rows at several scales: N(0.5, 3), with rows of variance ~1e-5 (where eps and the variance's divisor
    matter), rows whose mean is far above sigma (the mean's error carried through x - mu) and all-zero rows (y = b exactly)."""
    x = torch.randn(rows, C, generator=g) * 3 + 0.5
    x[1::7] *= 1e-3
    x[3::11] += 100.0
    x[5::13] = 0.0
    return x


def embed_x(ids, emb, pe, alpha, L):
    """The prologue's x (rows, C) in fp32: emb[clamp(id)] + alpha * pe[row % L]."""
    rows = ids.shape[0]
    return emb[ids.clamp(0, emb.shape[0] - 1)] + alpha * pe[torch.arange(rows) % L]


def bert_x(ids, tts, word, typ, pos, N):
    """BertEmbeddings' sum (rows, C) in fp32: (word[id] + type[tt]) + pos[row % N]."""
    return (word[ids] + typ[tts]) + pos[torch.arange(ids.shape[0]) % N]


def tracks(p, e, pros):
    """The pitch / energy tracks (T,) the convolutions read, after the fp32 prosody affine (pros: 5 floats or None)."""
    if pros is None:
        return p, e
    return p * pros[1] + pros[2], e * pros[3] + pros[4]


def var_embed_ref(x, p, e, wp, bp, we, be, pros, tl):
    """One item: x (T, C), tracks p / e (T,), taps wp / we (K, C), window clipped to [0, tl).  -> (y, m), each (T, C)."""
    T = x.shape[0]
    K = wp.shape[0]
    h = (K - 1) // 2
    p1, e1 = tracks(p, e, pros)
    y, m = x.double().clone(), x.double().abs()
    for tr, w_, b_ in ((p1, wp, bp), (e1, we, be)):
        pad = torch.zeros(T + 2 * h, dtype=torch.float64)
        pad[h:h + tl] = tr[:tl].double()
        win = pad.unfold(0, K, 1)                                   # (T, K): taps t - h .. t + h
        y = y + (win @ w_.double() + b_.double())
        m = m + win.abs() @ w_.double().abs() + b_.double().abs()
    return y, m


def gauss_ref(hs, c, tlen, frames, pe=None, alpha=None, chunk=64):
    """One item: hs (T, H), centres c (T,) fp32, the frames to compute (LongTensor).  -> (y, m), each (len(frames), H)."""
    h = hs[:tlen].double()
    cd = c[:tlen].double()
    f = frames.double()[:, None]
    e = -TENTH32 * (f - cd[None]) ** 2
    p = torch.softmax(e, -1)
    o = p @ h
    m = p @ h.abs()
    pe_ = p * e.abs()
    for i0 in range(0, len(frames), chunk):
        i1 = min(i0 + chunk, len(frames))
        m[i0:i1] += (pe_[i0:i1, :, None] * (h[None] - o[i0:i1, None]).abs()).sum(1)
    if pe is not None:
        ap = (alpha * pe[frames]).double()        # fp32 product, as the kernel rounds it
        o, m = o + ap, m + ap.abs()
    return o, m


def attn_check(out, qkv, klen, heads):
    """Every query row of one item (L, H) against fp64 over the keys j < klen (am_ref.attn_ref, score term included)."""
    y64, m = am_ref.attn_ref(qkv, klen, heads, rows=torch.arange(qkv.shape[0]))
    return check(out, y64, m)


def durations_expected(s64, m):
    """-> (d, d_lo, d_hi) per row: the fp64 duration and the range a kernel within the bound may return."""
    band = TAU * m
    d = torch.round(torch.exp(s64) - 1).clamp_min(0)
    d_lo = torch.round(torch.exp(s64 - band) * (1 - EXP_ULPS) - 1).clamp_min(0)
    d_hi = torch.round(torch.exp(s64 + band) * (1 + EXP_ULPS) - 1).clamp_min(0)
    return d, d_lo, d_hi


def check_rowdot(out, s64, m, valid, mode):
    """out (B, T) of a predictor head (float for mode 0, int64 durations for mode 1), s64 / m (B, T) from gemv_ref; valid =
    item lengths.  Pad rows must be exact zeros.  -> dict(ok, err_m, pads_zero, n_ambiguous, rows)."""
    B, T = out.shape
    vm = torch.arange(T)[None, :] < torch.tensor(valid)[:, None]
    pads_zero = bool((out[~vm] == 0).all())
    if mode == 0:
        r = check(out[vm], s64[vm], m[vm])
        return dict(r, ok=r["ok"] and pads_zero, pads_zero=pads_zero, n_ambiguous=0, rows=int(vm.sum()))
    d, lo, hi = durations_expected(s64[vm], m[vm])
    got = out[vm].double()
    inside = bool(((got >= lo) & (got <= hi)).all())
    amb = int((lo != hi).sum())
    return dict(ok=inside and pads_zero, err_m=0.0, pads_zero=pads_zero, in_band=inside, n_ambiguous=amb, rows=int(vm.sum()),
                n_off_fp64=int((got != d).sum()))


def find_ties(exp_fn, targets=(0.5, 2.5), span=4096):
    """fp32 s with fl32(exp_fn(s)) - 1 == v exactly, for each v in targets (None where the sweep of `span` consecutive fp32
    values around ln(v + 1) finds none).  exp_fn computes torch.exp on the device the kernel runs on."""
    out = {}
    for v in targets:
        s0 = torch.tensor(math.log(v + 1.0), dtype=torch.float32)
        bits = s0.view(torch.int32) + torch.arange(-span // 2, span // 2, dtype=torch.int32)
        s = bits.view(torch.float32)
        hit = ((exp_fn(s) - 1.0) == v).nonzero()
        out[v] = float(s[hit[0, 0]]) if hit.numel() else None
    return out


# ---- launch rules (am_kernels.cu) ---------------------------------------------------------------------------------------------
def ln_inst(C):
    """layernorm_kernel<NV>: NV = C / 128."""
    return ("layernorm", C // 128)


def attn_inst(B, L, H, heads, sms):
    """launch_attention: 32-query tiles while ceil(L / 64) * heads * B < 2 * SMs, 64-query tiles otherwise."""
    small = (L + 63) // 64 * heads * B < 2 * sms
    return ("attention", H // heads, 32 if small else 64)


def gauss_inst(B, F, H, sms):
    """launch_gauss_upsample: NC = H / 128; 8-frame tiles while B * ceil(F / 16) < 2 * SMs, 16-frame tiles otherwise."""
    small = B * ((F + 15) // 16) < 2 * sms
    return ("gauss", H // 128, 8 if small else 16)


# the instantiations a shipped configuration launches: LayerNorm at 256 (the small style encoder), 384 (the acoustic model) and
# 768 (BERT-base); FFMA attention at d_k = 48 (the "fp32_ffma" acoustic model) and 64 (both style encoders); Gaussian upsampling
# at H = 384
SHIPPED = {("layernorm", 2), ("layernorm", 3), ("layernorm", 6), ("attention", 48, 32), ("attention", 48, 64),
           ("attention", 64, 32), ("attention", 64, 64), ("gauss", 3, 8), ("gauss", 3, 16)}

# ---- operator cases -------------------------------------------------------------------------------------------------------------
H, HEADS, BERT, COND_K, K_EMBED = 384, 8, 768, 1920, 9
STYLE = ((256, 4), (768, 12))        # (hidden, heads) of the small and the full style encoder
EDGE_KLEN = (1, 63, 64, 65, 127, 128, 129)
EDGE_TLEN = (1, 15, 16, 17)


def corpus_lens(n=32):
    from emotivoice_b200 import synth
    return synth.corpus_lengths(n)


def points():
    """The acoustic tests' (name, item lengths): the headline B = 1 of 100 phonemes, b3_padded's (9, 23, 14) and 32 corpus
    utterances, with the edge lengths 1 / 8 / 9 / 15 / 16 / 17 in place of the first corpus items."""
    c = corpus_lens()
    return [("b1_t100", [100]), ("b3", [9, 23, 14]), ("b32", [max(c), 1, 8, 9, 15, 16, 17] + c[7:])]


def attn_cases():
    """(name, H, heads, item key lengths).  B = 1 picks 32-query tiles, the batches 64-query tiles (at 132 SMs).  "nomask"
    cases pass no key lengths, as the "fp32_ffma" decoder does for a literal batch."""
    cs = [("enc_b1_L100", H, HEADS, [100]), ("enc_b3", H, HEADS, [9, 23, 14]), ("dec_b1_L1100_nomask", H, HEADS, [1100]),
          ("enc_b32", H, HEADS, [200] + list(EDGE_KLEN) + corpus_lens()[8:])]
    for hid, hd in STYLE:
        cs.append(("sty%d_b1_L%d" % (hid, 128 if hid == 256 else 512), hid, hd, [128 if hid == 256 else 512]))
        B = 24 if hid == 256 else 8                       # ceil(129 / 64) * heads * B >= 264
        cs.append(("sty%d_b%d_L129" % (hid, B), hid, hd, list(EDGE_KLEN) + [(37 * i) % 129 + 1 for i in range(B - len(EDGE_KLEN))]))
    return cs


def gauss_cases():
    """(name, item token lengths, per-item total frames or None, per-item alpha).  Items with alpha 1 have their durations set
    so the frame count lands on the 8- / 16-frame tile edges; the others take fractional centres from the speaking rate."""
    c = corpus_lens()
    frames = [None, 8, 15, 16, 17, 31, 32, 33, 7]
    lens = [max(c), 1, 15, 16, 17, 16, 17, 33, 1] + c[9:]
    alphas = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0] + [0.5 + 0.05 * i for i in range(len(c) - 9)]
    return [("b1_t100", [100], [None], [1.25]), ("b1_t17", [17], [33], [1.0]),
            ("b3", [9, 23, 14], [None] * 3, [1.0, 0.8, 1.6]),
            ("b32", lens, frames + [None] * (len(c) - 9), alphas)]


def ln_cases():
    """(name, kernel, C, item lengths).  kernel: "ln" plain, "embed" the encoder's prologue, "bert" BertEmbeddings."""
    cs = []
    for name, lens in points():
        cs.append(("embed_" + name, "embed", H, lens))
        cs.append(("ln_" + name, "ln", H, lens))
    for hid, _ in STYLE:
        cs.append(("ln%d_b1" % hid, "ln", hid, [77]))
        cs.append(("ln%d_b5" % hid, "ln", hid, [77, 1, 9, 40, 13]))
        cs.append(("bert%d_b1" % hid, "bert", hid, [61]))
        cs.append(("bert%d_b3" % hid, "bert", hid, [61, 5, 33]))
    return cs


def case_instantiations(sms):
    """Every instantiation the cases launch at `sms` SMs (the B = 1 launches of each item included)."""
    inst = {ln_inst(C) for _, k, C, _ in ln_cases() if k != "bert"}
    for _, hid, hd, lens in attn_cases():
        inst.add(attn_inst(len(lens), max(lens), hid, hd, sms))
        inst |= {attn_inst(1, n, hid, hd, sms) for n in lens}
    for _, lens, frames, alphas in gauss_cases():
        F = est_frames(lens, frames, alphas)
        inst.add(gauss_inst(len(lens), max(F), H, sms))
        inst |= {gauss_inst(1, f, H, sms) for f in F}
    return inst


def durations_for(lens, frames, seed=11):
    """Integer durations (B, T) of the Gaussian cases: 1..9 per token, the last token's adjusted where `frames` fixes the
    item's total (alpha 1), zeros past each item."""
    g = torch.Generator().manual_seed(seed)
    B, T = len(lens), max(lens)
    d = torch.randint(1, 10, (B, T), generator=g)
    d[torch.arange(T)[None, :] >= torch.tensor(lens)[:, None]] = 0
    for b, (n, f) in enumerate(zip(lens, frames)):
        if f is not None:
            d[b, :n] = 0
            d[b, :n] = f // n
            d[b, n - 1] += f - int(d[b, :n].sum())
            assert d[b, :n].min() >= 0 and int(d[b].sum()) == f, (n, f)
    return d


def est_frames(lens, frames, alphas):
    """Per-item frame counts of the Gaussian cases (host side: trunc of the fp32 sum of fl32(d * alpha))."""
    d = durations_for(lens, frames)
    a = torch.tensor(alphas, dtype=torch.float32)
    return [int(torch.tensor(float((d[b].float() * a[b]).double().sum()), dtype=torch.float32)) for b in range(len(lens))]
