"""Host-only checks of tests/fp32_ref.py (no GPU): fp32 emulations of each kernel pass the fp64 check at TAU, and the check
rejects each of these seeded faults:

* LayerNorm with eps 1e-5, or with the unbiased variance; the prologue reading pe[row] instead of pe[row % L];
* cond_gemv with one 256-thread K slice dropped; row_gemv without its tanh; rowdot pads not zeroed; roundf on a tie row;
* var_embed_add with its taps mirrored, or with the prosody window ending at lens + 1 or at T;
* Gaussian upsampling dropping the last 16-token chunk, or normalising over T tokens instead of the item's tlen;
* attention admitting the key at klen, or dropping the key at klen - 1.

At 132 SMs (an H100 SXM) the operator cases launch every instantiation a shipped configuration uses.
"""
import math

import pytest
import torch

import fp32_ref as R


def test_cases_cover_every_shipped_instantiation_at_132_sms():
    inst = R.case_instantiations(132)
    assert R.SHIPPED <= inst, R.SHIPPED - inst
    assert R.attn_inst(1, 100, 384, 8, 132) == ("attention", 48, 32) and R.attn_inst(32, 200, 384, 8, 132) == ("attention", 48, 64)
    assert R.gauss_inst(1, 2000, 384, 132) == ("gauss", 3, 8) and R.gauss_inst(32, 700, 384, 132) == ("gauss", 3, 16)


# ---- LayerNorm ------------------------------------------------------------------------------------------------------------------
def _ln32(x, w, b, eps=1e-12, unbiased=False):
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = (d * d).sum(-1, keepdim=True) / (x.shape[-1] - (1 if unbiased else 0))
    return d * torch.rsqrt(var + eps) * w + b


@pytest.mark.parametrize("C", [256, 384, 768])
def test_layernorm_faults(C):
    g = torch.Generator().manual_seed(C)
    x = R.ln_input(100, C, g)
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    assert R.ln_check(_ln32(x, w, b), x, w, b)["ok"]
    assert not R.ln_check(_ln32(x, w, b, eps=1e-5), x, w, b)["ok"]
    assert not R.ln_check(_ln32(x, w, b, unbiased=True), x, w, b)["ok"]


def test_prologue_pe_row_fault():
    g = torch.Generator().manual_seed(5)
    B, L, C = 3, 23, 384
    emb, w, b = torch.randn(50, C, generator=g), torch.randn(C, generator=g), torch.randn(C, generator=g)
    pe = torch.randn(B * L, C, generator=g)
    ids = torch.randint(0, 50, (B * L,), generator=g)
    alpha = torch.tensor([1.7])
    x = R.embed_x(ids, emb, pe, alpha, L)
    assert R.ln_check(_ln32(x, w, b), x, w, b)["ok"]
    bad = emb[ids] + alpha * pe[torch.arange(B * L)]
    assert not R.ln_check(_ln32(bad, w, b), x, w, b)["ok"]


# ---- GEMVs and the predictor heads ------------------------------------------------------------------------------------------------
def test_cond_gemv_dropped_k_slice():
    g = torch.Generator().manual_seed(7)
    c = torch.randn(3, R.COND_K, generator=g)
    w, bias = torch.randn(R.COND_K, R.H, generator=g) / math.sqrt(R.COND_K), torch.randn(R.H, generator=g)
    y64, m = R.gemv_ref(c, w, bias)
    assert R.check(c @ w + bias, y64, m)["ok"]
    keep = torch.ones(R.COND_K)
    keep[3 * 256:4 * 256] = 0                     # the fourth pass of the 256 threads over K
    assert not R.check((c * keep) @ w + bias, y64, m)["ok"]


def test_row_gemv_missing_tanh():
    g = torch.Generator().manual_seed(8)
    x, w, bias = torch.randn(6, 768, generator=g), torch.randn(768, 768, generator=g) * (1.5 / math.sqrt(768)), torch.randn(768, generator=g)
    y64, m = R.gemv_ref(x, w, bias, tanh=True)
    assert R.check(torch.tanh(x @ w + bias), y64, m)["ok"]
    assert not R.check(x @ w + bias, y64, m)["ok"]


def _heads_case():
    g = torch.Generator().manual_seed(9)
    lens = [23, 9, 14]
    B, T, C = 3, 23, R.H
    x = torch.randn(B, T, C, generator=g)
    w = torch.randn(C, generator=g) * (0.6 / math.sqrt(C))
    bias = torch.tensor([1.2])
    s64, m = R.gemv_ref(x.reshape(B * T, C), w[:, None], bias)
    s32 = (x @ w + bias).reshape(B, T)
    return lens, s32, s64.reshape(B, T), m.reshape(B, T)


@pytest.mark.parametrize("mode", [0, 1])
def test_rowdot_pads_not_zeroed(mode):
    lens, s32, s64, m = _heads_case()
    out = s32 if mode == 0 else torch.round(torch.exp(s32) - 1).clamp_min(0).long()
    vm = torch.arange(s32.shape[1])[None, :] < torch.tensor(lens)[:, None]
    good = torch.where(vm, out, torch.zeros_like(out))
    r = R.check_rowdot(good, s64, m, lens, mode)
    assert r["ok"] and r["n_ambiguous"] <= max(1, r["rows"] // 100), r
    assert not R.check_rowdot(out, s64, m, lens, mode)["ok"]


def test_duration_tie_rint_not_roundf():
    ties = R.find_ties(torch.exp, targets=(0.5,))
    s = torch.tensor([ties[0.5]], dtype=torch.float32)
    v = torch.exp(s) - 1
    assert float(v) == 0.5
    assert int(torch.round(v)) == 0                 # rint: half to even, what the duration must be
    assert int(torch.floor(v + 0.5)) != 0           # roundf (half away from zero) fails the tie assertion
    # the generic check accepts either neighbour of a tie (the fp64 exp lies within the band)
    _, lo, hi = R.durations_expected(s.double(), s.double().abs())
    assert int(lo) == 0 and int(hi) == 1


# ---- var_embed_add --------------------------------------------------------------------------------------------------------------
def _var_embed32(x, p, e, wp, bp, we, be, pros, tl):
    T = x.shape[0]
    K = wp.shape[0]
    h = (K - 1) // 2
    p1, e1 = R.tracks(p, e, pros)
    y = []
    for tr, w_, b_ in ((p1, wp, bp), (e1, we, be)):
        pad = torch.zeros(T + 2 * h)
        pad[h:h + tl] = tr[:tl]
        y.append(pad.unfold(0, K, 1) @ w_ + b_)
    return (x + y[0]) + y[1]


@pytest.mark.parametrize("fault", ["mirrored_taps", "window_lens_plus_1", "window_T"])
def test_var_embed_faults(fault):
    g = torch.Generator().manual_seed(10)
    T, n, C, K = 30, 21, R.H, R.K_EMBED
    x, p, e = torch.randn(T, C, generator=g), torch.randn(T, generator=g), torch.randn(T, generator=g)
    p[n - 1], e[n - 1], p[n], e[n] = 40.0, -30.0, 1e3, -1e3         # large at the last token and the first pad
    wp, we = torch.randn(K, C, generator=g) / 3, torch.randn(K, C, generator=g) / 3
    bp, be = torch.randn(C, generator=g), torch.randn(C, generator=g)
    pros = torch.tensor([1.0, 1.3, 0.4, 0.7, -0.2])
    y64, m = R.var_embed_ref(x, p, e, wp, bp, we, be, pros, n)
    assert R.check(_var_embed32(x, p, e, wp, bp, we, be, pros, n), y64, m)["ok"]
    if fault == "mirrored_taps":
        bad = _var_embed32(x, p, e, wp.flip(0), bp, we.flip(0), be, pros, n)
    else:
        bad = _var_embed32(x, p, e, wp, bp, we, be, pros, n + 1 if fault == "window_lens_plus_1" else T)
    assert not R.check(bad, y64, m)["ok"]


# ---- Gaussian upsampling -------------------------------------------------------------------------------------------------------
def _centres(d, alpha):
    ds = d.float() * alpha
    return (torch.cumsum(ds.double(), 0).float() - ds * 0.5), ds


def _gauss32(hs, c, tlen, frames, norm_tokens=None, drop_from=None):
    f = frames.float()[:, None]
    nt = norm_tokens or tlen
    e = -0.1 * (f - c[None, :nt]) ** 2
    p = torch.softmax(e, -1)[:, :tlen]
    if drop_from is not None:
        p = p.clone()
        p[:, drop_from:] = 0
    return p @ hs[:tlen]


@pytest.mark.parametrize("fault", ["last_chunk_dropped", "normalised_over_T"])
def test_gauss_faults(fault):
    g = torch.Generator().manual_seed(11)
    T, tlen, H = 24, 17, R.H
    d = torch.randint(1, 8, (T,), generator=g)
    d[tlen:] = 0
    c, ds = _centres(d, torch.tensor(0.8))
    F = int(float(ds.double().sum()))
    hs = torch.randn(T, H, generator=g)
    frames = torch.arange(F)
    y64, m = R.gauss_ref(hs, c, tlen, frames)
    assert R.check(_gauss32(hs, c, tlen, frames), y64, m)["ok"]
    if fault == "last_chunk_dropped":
        bad = _gauss32(hs, c, tlen, frames, drop_from=(tlen - 1) // 16 * 16)
    else:
        bad = _gauss32(hs, c, tlen, frames, norm_tokens=T)
    assert not R.check(bad, y64, m)["ok"]


# ---- attention ----------------------------------------------------------------------------------------------------------------
def _attn32(qkv, nkeys, heads):
    L, H3 = qkv.shape
    H = H3 // 3
    dk = H // heads
    q, k, v = [t.reshape(L, heads, dk).transpose(0, 1) for t in qkv.split(H, -1)]
    p = torch.softmax(q @ k[:, :nkeys].transpose(1, 2) / math.sqrt(dk), -1)
    return (p @ v[:, :nkeys]).transpose(0, 1).reshape(L, H)


@pytest.mark.parametrize("hid,heads", R.STYLE + ((R.H, R.HEADS),))
def test_attention_key_edge_faults(hid, heads):
    g = torch.Generator().manual_seed(hid)
    L, klen = 129, 65
    qkv = torch.randn(L, 3 * hid, generator=g)
    assert R.attn_check(_attn32(qkv, klen, heads), qkv, klen, heads)["ok"]
    assert not R.attn_check(_attn32(qkv, klen + 1, heads), qkv, klen, heads)["ok"]
    assert not R.attn_check(_attn32(qkv, klen - 1, heads), qkv, klen, heads)["ok"]
