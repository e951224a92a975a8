"""The fp32 kernels between the acoustic model's GEMMs and the style encoder's own kernels against fp64, at the engine's shapes
and instantiations, with item lengths on the kernels' edges.

References, magnitudes, launch rules and cases: tests/fp32_ref.py.  Every valid output element must satisfy |y - y64| <= TAU * m
(TAU = 2^-14), and each result REL_MAX of max|y64|.  Durations must lie in the range the bound allows (either neighbour where it
straddles a rounding boundary).  Besides the bound:

* never read: the K and V thirds of qkv rows >= klen, hs rows and centres past an item's tokens and the pad rows of the predictor
  heads' and mask_rows' input are NaN; pad rows of rowdot and mask_rows must come out as exact zeros;
* exact zeros: Gaussian frames >= mel_lens[b] under the batch-invariant contract; an all-zero LayerNorm row gives exactly b;
* bitwise: each item of a ragged batch equals its own batch-1 launch (for attention and Gaussian upsampling the batch-1 launch
  takes the small tile and the batch the large one); the prologue's x equals torch's fp32 emb[id] + alpha * pe[t] (out-of-range
  ids read the clamped row); prosody (alpha, 1, 0, 1, 0) equals no prosody.

Largest err/m measured on an H100 80GB HBM3 (132 SMs, 700 W power limit):
    layernorm 2^-22.9   layernorm_embed 2^-23.2   bert_embed_ln 2^-23.1   cond_gemv 2^-25.2   row_gemv 2^-24.6   rowdot 2^-24.7
    var_embed_add 2^-22.4   gauss_upsample 2^-21.8   attention d_k 48 2^-22.4   attention d_k 64 2^-22.5
Durations: 13 of the batch of 32's 3198 rows lie in the ambiguity band, none of the B = 1 and B = 3 rows; every duration equals
its fp64 value.  Both half-even ties were found on the device (exp(s) - 1 = 0.5 at s = 0.405465096, 2.5 at s = 1.25276291) and
gave 0 and 2.  The whole file took 12 s.
"""
import math

import pytest
import torch

import fp32_ref as R
from emotivoice_b200 import _abi, packing

pytestmark = pytest.mark.gpu
WORST = {}


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _run(rc):
    _abi.check(rc)
    torch.cuda.synchronize()


def _same(a, b):
    a, b = a.contiguous().cpu(), b.contiguous().cpu()
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return a.shape == b.shape and torch.equal(a, b)


def _record(kernel, r, what=""):
    WORST[kernel] = max(WORST.get(kernel, 0.0), r["err_m"])
    assert r["ok"], (kernel, what, r)


def _nan_rows_past(t, lens):
    t = t.clone()
    for b, n in enumerate(lens):
        t[b, n:] = float("nan")
    return t


def test_cases_launch_every_shipped_instantiation():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    inst = R.case_instantiations(sms)
    print("SMs %d, instantiations launched: %s" % (sms, sorted(inst)))
    assert R.SHIPPED <= inst, R.SHIPPED - inst


# ---- LayerNorm: plain, with the encoder's embedding prologue, BertEmbeddings -------------------------------------------------
@pytest.mark.parametrize("case", R.ln_cases(), ids=[c[0] for c in R.ln_cases()])
def test_layernorm(lib, dev, case):
    name, kind, C, lens = case
    B, T = len(lens), max(lens)
    rows = B * T
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    wd, bd = w.to(dev), b.to(dev)
    y = torch.full((rows, C), float("nan"), device=dev)
    if kind == "ln":
        x = R.ln_input(rows, C, g)
        xd = x.to(dev)

        def launch(x_, y_, n_rows, L):
            return lib.ev_op_layernorm(_p(x_), _p(wd), _p(bd), _p(y_), n_rows, C, _st())
        _run(launch(xd, y, rows, T))
        x32 = x
        zero = (x == 0).all(1)
        assert zero.any() and _same(y.cpu()[zero], b.expand(int(zero.sum()), C))
    elif kind == "embed":
        n_emb = 300
        emb = torch.randn(n_emb, C, generator=g)
        pe = packing.build_pe_table(T, C)
        alpha = torch.tensor([1.7])
        ids = torch.randint(0, n_emb, (B, T), generator=g)
        ids[0, 0], ids[-1, min(1, T - 1)] = n_emb + 9, -3        # out of range: the kernel reads the clamped row
        ed, ped, ad = emb.to(dev), pe.to(dev), alpha.to(dev)
        x_out = torch.full((rows, C), float("nan"), device=dev)
        idd = ids.to(dev)

        def launch(ids_, y_, n_rows, L, x_out_=None):
            return lib.ev_op_layernorm_embed(_p(ids_), _p(ed), n_emb, _p(ped), _p(ad), L, _p(x_out_), _p(wd), _p(bd), _p(y_), n_rows, C,
                                             _st())
        _run(launch(idd, y, rows, T, x_out))
        x32 = R.embed_x(ids.reshape(-1), emb, pe, alpha, T)
        assert _same(x_out, x32)
    else:
        vocab, N = 1000, T
        word, typ = torch.randn(vocab, C, generator=g) * 0.5, torch.randn(2, C, generator=g) * 0.5
        pos = torch.randn(max(T, 128), C, generator=g) * 0.5
        ids = torch.randint(0, vocab, (B, T), generator=g)
        tts = torch.randint(0, 2, (B, T), generator=g)
        wdv, td, pd = word.to(dev), typ.to(dev), pos.to(dev)
        idd, ttd = ids.to(dev), tts.to(dev)

        def launch(ids_, y_, n_rows, L, tts_=None):
            return lib.ev_op_bert_embed_ln(_p(ids_), _p(tts_), _p(wdv), _p(td), _p(pd), _p(wd), _p(bd), _p(y_), n_rows, L, C, _st())
        _run(launch(idd, y, rows, N, ttd))
        x32 = R.bert_x(ids.reshape(-1), tts.reshape(-1), word, typ, pos, N)
    _record("bert_embed_ln" if kind == "bert" else "layernorm" + ("_embed" if kind == "embed" else ""), R.ln_check(y.cpu(), x32, w, b), name)
    if B > 1:
        yb = y.reshape(B, T, C)
        for i, n in enumerate(lens):
            y1 = torch.full((n, C), float("nan"), device=dev)
            if kind == "ln":
                _run(launch(xd[i * T:i * T + n].contiguous(), y1, n, n))
            elif kind == "embed":
                x1 = torch.full((n, C), float("nan"), device=dev)
                _run(launch(idd[i, :n].contiguous(), y1, n, n, x1))
                assert _same(x1, x_out.reshape(B, T, C)[i, :n]), (name, i)
            else:
                _run(launch(idd[i, :n].contiguous(), y1, n, n, ttd[i, :n].contiguous()))
            assert _same(y1, yb[i, :n]), (name, i, n)


# ---- FFMA attention -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", R.attn_cases(), ids=[c[0] for c in R.attn_cases()])
def test_attention(lib, dev, case):
    name, hid, heads, lens = case
    B, L = len(lens), max(lens)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    qkv = torch.randn(B, L, 3 * hid, generator=g)
    for b, n in enumerate(lens):
        qkv[b, n:, hid:] = float("nan")            # keys and values past klen are never read; the queries there are computed
    qd = qkv.to(dev)
    ld = None if name.endswith("nomask") else torch.tensor(lens, dtype=torch.int32, device=dev)
    out = torch.full((B, L, hid), float("nan"), device=dev)
    _run(lib.ev_op_attention(_p(qd), _p(ld), _p(out), B, L, hid, heads, _st()))
    got = out.cpu()
    for b, n in enumerate(lens):
        _record("attention_dk%d" % (hid // heads), R.attn_check(got[b], qkv[b], n, heads), (name, b, n))
    if B > 1:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert B < 8 or R.attn_inst(B, L, hid, heads, sms)[2] == 64      # the batches of 8 and more take the large tile
        for b, n in enumerate(lens):
            assert R.attn_inst(1, n, hid, heads, sms)[2] == 32
            q1 = qd[b:b + 1, :n].contiguous()
            o1 = torch.full((1, n, hid), float("nan"), device=dev)
            _run(lib.ev_op_attention(_p(q1), None, _p(o1), 1, n, hid, heads, _st()))
            assert _same(o1[0], out[b, :n]), (name, b, n)


# ---- Gaussian upsampling -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", R.gauss_cases(), ids=[c[0] for c in R.gauss_cases()])
def test_gauss_upsample(lib, dev, case):
    name, lens, frames, alphas = case
    B, T = len(lens), max(lens)
    d = R.durations_for(lens, frames)
    dd, ld = d.to(dev), torch.tensor(lens, dtype=torch.int32, device=dev)
    ad = torch.tensor(alphas, dtype=torch.float32, device=dev)
    centers = torch.empty(B, T, device=dev)
    ds = torch.empty(B, T, device=dev)
    mel = torch.empty(B + 1, dtype=torch.int32, device=dev)
    _run(lib.ev_op_duration_scan(_p(dd), _p(ld), _p(ad), 1, B, T, _p(centers), _p(ds), _p(mel), _st()))
    ml = mel.cpu()[:B].tolist()
    F = int(mel[B])
    assert ml == R.est_frames(lens, frames, alphas)
    for b, (n, f) in enumerate(zip(lens, frames)):
        assert f is None or ml[b] == f
        centers[b, n:] = float("nan")
    c = centers.cpu()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    hs = _nan_rows_past(torch.randn(B, T, R.H, generator=g), lens)
    hd = hs.to(dev)
    pe = packing.build_pe_table(F, R.H)
    dec_alpha = torch.tensor([1.3])
    ped, dad = pe.to(dev), dec_alpha.to(dev)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for invariant in ((1, 0) if name == "b3" else (1,)):
        out = torch.full((B, F, R.H), float("nan"), device=dev)
        _run(lib.ev_op_gauss_upsample_centers(_p(hd), _p(centers), _p(ld), _p(mel), B, T, R.H, F, invariant, _p(ped), _p(dad), _p(out),
                                              _st()))
        got = out.cpu()
        for b, n in enumerate(lens):
            fl = ml[b] if invariant else F
            y64, m = R.gauss_ref(hs[b], c[b], n, torch.arange(fl), pe, dec_alpha)
            _record("gauss_upsample", R.check(got[b, :fl], y64, m), (name, invariant, b, n, fl))
            assert bool((got[b, fl:] == 0).all()), (name, b)
    if B > 1:
        assert B < 8 or R.gauss_inst(B, F, R.H, sms)[2] == 16
        for b, n in enumerate(lens):
            fl = ml[b]
            assert R.gauss_inst(1, fl, R.H, sms)[2] == 8
            o1 = torch.full((1, fl, R.H), float("nan"), device=dev)
            h1, c1 = hd[b:b + 1, :n].contiguous(), centers[b:b + 1, :n].contiguous()
            l1, m1 = torch.tensor([n], dtype=torch.int32, device=dev), torch.tensor([fl], dtype=torch.int32, device=dev)
            _run(lib.ev_op_gauss_upsample_centers(_p(h1), _p(c1), _p(l1), _p(m1), 1, n, R.H, fl, 1, _p(ped), _p(dad), _p(o1), _st()))
            assert _same(o1[0], out[b, :fl]), (name, b, n, fl)


# ---- pitch / energy embedding ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pt", R.points(), ids=[p[0] for p in R.points()])
def test_var_embed_add(lib, dev, pt):
    name, lens = pt
    B, T, C, K = len(lens), max(lens), R.H, R.K_EMBED
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 5)
    x = torch.randn(B, T, C, generator=g)
    p, e = torch.randn(B, T, generator=g), torch.randn(B, T, generator=g)
    for b, n in enumerate(lens):
        p[b, n - 1], e[b, n - 1] = 40.0, -30.0                       # large at the last token ...
        p[b, n:] = 1e3 * (1 + torch.rand(T - n, generator=g))         # ... and garbage in the pads
        e[b, n:] = -1e3 * (1 + torch.rand(T - n, generator=g))
    wp, we = torch.randn(K, C, generator=g) / 3, torch.randn(K, C, generator=g) / 3
    bp, be = torch.randn(C, generator=g), torch.randn(C, generator=g)
    pros = torch.stack([torch.tensor([1.0, 1.3 - 0.1 * b, 0.4 + 0.05 * b, 0.7, -0.2 - 0.01 * b]) for b in range(B)])
    xd, pd_, ed = x.to(dev), p.to(dev), e.to(dev)
    wpd, wed, bpd, bed = wp.to(dev), we.to(dev), bp.to(dev), be.to(dev)
    ld, prd = torch.tensor(lens, dtype=torch.int32, device=dev), pros.to(dev)

    def launch(x_, p_, e_, pr_, l_, B_, T_):
        y = x_.clone()
        _run(lib.ev_op_var_embed_add(_p(y), _p(p_), _p(e_), _p(wpd), _p(bpd), _p(wed), _p(bed), _p(pr_), _p(l_), B_, T_, C, K, _st()))
        return y

    plain = launch(xd, pd_, ed, None, None, B, T).cpu()           # no prosody: the window ends at T, pads are data
    shaped = launch(xd, pd_, ed, prd, ld, B, T)                    # prosody with lens: the window ends at lens[b]
    got = shaped.cpu()
    for b, n in enumerate(lens):
        y64, m = R.var_embed_ref(x[b], p[b], e[b], wp, bp, we, be, None, T)
        _record("var_embed_add", R.check(plain[b], y64, m), (name, "plain", b))
        y64, m = R.var_embed_ref(x[b], p[b], e[b], wp, bp, we, be, pros[b], n)
        _record("var_embed_add", R.check(got[b], y64, m), (name, "prosody", b))
        one = launch(xd[b:b + 1, :n].contiguous(), pd_[b:b + 1, :n].contiguous(), ed[b:b + 1, :n].contiguous(), prd[b:b + 1].contiguous(),
                     ld[b:b + 1].contiguous(), 1, n)
        assert _same(one[0], shaped[b, :n]), (name, b, n)
    neutral = torch.tensor([[1.0, 1.0, 0.0, 1.0, 0.0]] * B, device=dev)
    full = torch.full((B,), T, dtype=torch.int32, device=dev)
    assert _same(launch(xd, pd_, ed, neutral, full, B, T), plain)


# ---- predictor heads, durations, mask_rows ------------------------------------------------------------------------------------
@pytest.mark.parametrize("pt", R.points(), ids=[p[0] for p in R.points()])
def test_rowdot_and_durations(lib, dev, pt):
    name, lens = pt
    B, T, C = len(lens), max(lens), R.H
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 9)
    x = _nan_rows_past(torch.randn(B, T, C, generator=g), lens)
    w = torch.randn(C, generator=g) * (0.6 / math.sqrt(C))
    bias = torch.tensor([1.2])
    xd, wd, bd, ld = x.to(dev), w.to(dev), bias.to(dev), torch.tensor(lens, dtype=torch.int32, device=dev)
    xs = torch.nan_to_num(x, nan=0.0).reshape(B * T, C)
    s64, m = R.gemv_ref(xs, w[:, None], bias)
    s64, m = s64.reshape(B, T), m.reshape(B, T)
    outs = {}
    for mode in (0, 1):
        out = (torch.full((B, T), float("nan"), device=dev) if mode == 0 else torch.full((B, T), -7, dtype=torch.int64, device=dev))
        _run(lib.ev_op_rowdot(_p(xd), _p(wd), _p(bd), _p(ld), B, T, C, mode, _p(out) if mode == 0 else None,
                              _p(out) if mode == 1 else None, _st()))
        outs[mode] = out
        r = R.check_rowdot(out.cpu(), s64, m, lens, mode)
        if mode == 0:
            _record("rowdot", r, name)
        else:
            print("%s durations: %d rows, %d in the ambiguity band, %d off the fp64 value" % (name, r["rows"], r["n_ambiguous"],
                                                                                              r["n_off_fp64"]))
            assert r["ok"], r
            assert r["n_ambiguous"] <= max(1, r["rows"] // 100), r
        for b, n in enumerate(lens):
            o1 = torch.full_like(out[b:b + 1, :n], -7) if mode == 1 else torch.full((1, n), float("nan"), device=dev)
            _run(lib.ev_op_rowdot(_p(xd[b:b + 1, :n].contiguous()), _p(wd), _p(bd), _p(ld[b:b + 1].contiguous()), 1, n, C, mode,
                                  _p(o1) if mode == 0 else None, _p(o1) if mode == 1 else None, _st()))
            assert _same(o1[0], out[b, :n]), (name, mode, b)
    # mask_rows: the literal batch's predictor input
    y = torch.full((B, T, C), 7.0, device=dev)
    _run(lib.ev_op_mask_rows(_p(xd), _p(ld), _p(y), B, T, C, _st()))
    for b, n in enumerate(lens):
        assert _same(y[b, :n], xd[b, :n]) and bool((y[b, n:] == 0).all()), (name, b)
        y1 = torch.full((1, n, C), 7.0, device=dev)
        _run(lib.ev_op_mask_rows(_p(xd[b:b + 1, :n].contiguous()), _p(ld[b:b + 1].contiguous()), _p(y1), 1, n, C, _st()))
        assert _same(y1[0], y[b, :n])
    y = torch.full((B, T, C), 7.0, device=dev)
    _run(lib.ev_op_mask_rows(_p(xd), None, _p(y), B, T, C, _st()))
    assert _same(y, xd)


def _duration_rows(lib, dev, s):
    """Durations of rows whose only non-zero channel is s (x = s, w = 1, bias 0): the kernel's s is exactly that fp32 value."""
    C = R.H
    x = torch.zeros(1, len(s), C)
    x[0, :, 0] = torch.tensor(s, dtype=torch.float32)
    w = torch.zeros(C)
    w[0] = 1.0
    xd, wd, bd = x.to(dev), w.to(dev), torch.zeros(1, device=dev)
    out = torch.full((1, len(s)), -7, dtype=torch.int64, device=dev)
    _run(lib.ev_op_rowdot(_p(xd), _p(wd), _p(bd), None, 1, len(s), C, 1, None, _p(out), _st()))
    return out.cpu()[0], x[0, :, 0].double()


def test_duration_edges(lib, dev):
    """Rows far below 0 (d = 0) and just either side of every rounding boundary ln(k + 1.5), k = 0..8."""
    s = [-20.0, -3.0, -0.1]
    for k in range(9):
        s += [math.log(k + 1.5) - 1e-3, math.log(k + 1.5) + 1e-3]
    d, s32 = _duration_rows(lib, dev, s)
    want, lo, hi = R.durations_expected(s32, s32.abs())
    assert torch.equal(lo, hi)                       # no row of this set is ambiguous
    assert d.tolist() == want.long().tolist()
    assert d[:3].tolist() == [0, 0, 0] and d[3::2].tolist() == list(range(9)) and d[4::2].tolist() == list(range(1, 10))


@pytest.mark.parametrize("v,want", [(0.5, 0), (2.5, 2)])
def test_duration_half_even_ties(lib, dev, v, want):
    """s where fl32(exp(s)) - 1 is exactly v: rint rounds the tie to even (torch.round semantics), roundf would not."""
    ties = R.find_ties(lambda t: torch.exp(t.to(dev)).cpu(), targets=(v,))
    if ties[v] is None:
        pytest.skip("no fp32 s near ln(%g) has exp(s) - 1 == %g exactly on this device: the tie cannot be posed" % (v + 1, v))
    d, _ = _duration_rows(lib, dev, [ties[v]])
    print("tie s = %.9g: d = %d" % (ties[v], int(d[0])))
    assert int(d[0]) == want


# ---- conditioning bias ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pt", R.points(), ids=[p[0] for p in R.points()])
def test_cond_bias(lib, dev, pt):
    name, lens = pt
    B, Hh, bert, n_spk = len(lens), R.H, R.BERT, 50
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 13)
    spk_emb = torch.randn(n_spk, Hh, generator=g)
    style, content = torch.randn(B, bert, generator=g), torch.randn(B, bert, generator=g)
    w = torch.randn(R.COND_K, Hh, generator=g) / math.sqrt(R.COND_K)
    bias = torch.randn(Hh, generator=g)
    spk = torch.randint(0, n_spk, (B,), generator=g)
    spk[0] = n_spk + 9                                            # out of range: the clamped row
    dv = [t.to(dev) for t in (spk, spk_emb, style, content, w, bias)]

    def launch(B_, sl):
        ci = torch.full((B_, R.COND_K), float("nan"), device=dev)
        o = torch.full((B_, Hh), float("nan"), device=dev)
        _run(lib.ev_op_cond_bias(_p(dv[0][sl].contiguous()), _p(dv[1]), n_spk, _p(dv[2][sl].contiguous()), _p(dv[3][sl].contiguous()), B_,
                                 Hh, bert, _p(dv[4]), _p(dv[5]), _p(ci), _p(o), _st()))
        return ci, o

    ci, out = launch(B, slice(0, B))
    c32 = R.cond_input(spk, spk_emb, style, content)
    assert _same(ci, c32)
    y64, m = R.gemv_ref(c32, w, bias)
    _record("cond_gemv", R.check(out.cpu(), y64, m), name)
    for b in range(B):
        _, o1 = launch(1, slice(b, b + 1))
        assert _same(o1[0], out[b]), (name, b)


# ---- the style encoder's pooler and heads ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("hid", [h for h, _ in R.STYLE])
@pytest.mark.parametrize("kind", ["pooler", "heads"])
@pytest.mark.parametrize("B", [1, 6])
def test_row_gemv(lib, dev, hid, kind, B):
    g = torch.Generator().manual_seed(hid + B + len(kind))
    n_tok = 13
    if kind == "pooler":      # tanh(Wp x[CLS] + bp): x = row 0 of each item's (n_tok, hid) block
        x, stride, N, act = torch.randn(B, n_tok, hid, generator=g), n_tok * hid, hid, _abi.ACT_TANH
        xk = x[:, 0]
    else:                     # the packed classification heads on the pooled vector
        x, stride, N, act = torch.randn(B, hid, generator=g), hid, 16, _abi.ACT_NONE
        xk = x
    w = torch.randn(hid, N, generator=g) * (1.5 / math.sqrt(hid))
    bias = torch.randn(N, generator=g) * 0.5
    xd, wd, bd = x.to(dev), w.to(dev), bias.to(dev)
    out = torch.full((B, N), float("nan"), device=dev)
    _run(lib.ev_op_row_gemv(_p(xd), stride, _p(wd), _p(bd), _p(out), B, hid, N, act, _st()))
    y64, m = R.gemv_ref(xk, w, bias, tanh=(kind == "pooler"))
    _record("row_gemv", R.check(out.cpu(), y64, m), (hid, kind, B))
    for b in range(B):
        o1 = torch.full((1, N), float("nan"), device=dev)
        _run(lib.ev_op_row_gemv(_p(xd[b:b + 1].contiguous()), stride, _p(wd), _p(bd), _p(o1), 1, hid, N, act, _st()))
        assert _same(o1[0], out[b])


def test_zz_largest_err_over_m():
    """Prints the largest err/m each kernel reached in this session's cases."""
    print("largest err/m per kernel:", {k: "%.3g (2^%.1f)" % (v, math.log2(v) if v > 0 else -math.inf) for k, v in sorted(WORST.items())})
