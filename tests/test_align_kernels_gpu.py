"""The four kernels of csrc/align_kernels.cu through their C ABI (ev_op_mas, ev_op_average_by_duration, ev_op_align_logp,
ev_op_get_segments) and the Python wrappers, against the reference's own search and averages (tests/golden/mas_*, avg_*, made
by oracle/make_golden_align.py from the reference's numba functions) and against float64 restatements (oracle/align_oracle.py).

Bounds (u = 2^-24, the float32 unit roundoff):

* Monotonic alignment search: paths and durations are integers, identical to the reference.  The per-item loss is -mean_j of
  the float32 log_p along the path; the kernel sums it in float64 (F <= 1800 terms: error <= F 2^-53 of the sum of |terms|,
  far below a float32 ulp) and rounds once, so it is within 1 ulp of fl32(-mean64).

* Averaging: y = fl32(S / n) with S the float64 sum of n float32 values, so |y - fl32(mean64)| <= 1 ulp(fl32(mean64)) plus the
  float64 sum's n 2^-53 mean|x| (negligible at these n).  The reference's own float32 running sum deviates from mean64 by the
  fixture's stored `averaged_dev` (up to 3.75 ulp on the energy-like track), so against the reference the bound is
  1 ulp + n 2^-53 mean|x| + averaged_dev.  Measured on an H100 80GB HBM3 (700 W power limit): the kernel equals
  fl32(mean64) on every element of every case here (largest |y - fl32(mean64)| = 0 ulp).

* align_logp: one warp per frame, A = 32 lanes x NC float4 (NC = A / 128).  With s_t the score of token t, mx their maximum,
  lse = mx + log sum_t exp(s_t - mx) and tl the item's unmasked tokens:
    - the squared distance sums non-negative terms: a rounded difference (2u on its square), the product (u), two adds inside a
      float4, NC adds per lane and the 5-step shuffle tree: (NC + 10) u relative; sqrtf (correctly rounded) halves it and adds u:
      |ds_t| <= c_s u |s_t|, c_s = NC / 2 + 6;
    - the exp arguments s_t - mx are off by <= (c_s + 1) u (|s_t| + |mx|); weighted by the softmax this is <= (c_s + 1) u (2|mx|
      + ln tl), because sum_t w_t (mx - s_t) <= sum_t w_t (lse - s_t) = entropy <= ln tl; expf (2 ulp) adds 4u, the sum of tl
      non-negative terms (ceil(tl / 32) sequential per lane, then 5 levels) (ceil(tl / 32) + 5) u, logf 1 ulp of ln(sum) <= 2u ln tl,
      the final add u |lse|; and |mx| <= |lse| + ln tl because mx <= lse <= mx + ln tl and mx <= 0;
    - y = fl(fl(s_t - lse) + prior) adds u (|s_t| + |lse|) and u |y|.
  Collected: |y - y64| <= tau (|s64_t| + |lse64|) + kappa + 2^-24 |y64|, tau = (3 c_s + 4) u (28u at NC = 4),
  kappa = ((4 c_s + 5) ln tl + ceil(tl / 32) + 9) u.  kappa is the exp / sum / log chain: its errors are relative to the sum,
  which is >= 1, so they are absolute in log space and do not shrink with |s| + |lse|.  The -inf pattern is identical.
  Largest err / (|s64| + |lse64|) measured on an H100 80GB HBM3 (700 W power limit) over all T, F and text_lens cases:
      A=128 2^-22.7   A=256 2^-23.2   A=384 2^-23.1   A=512 2^-23.3      (tau: 2^-19.4 at NC = 1 to 2^-19.2 at NC = 4)
  AlignmentModule adds its five 3xTF32 convolutions: each output is within 2^-14 of the sum of the magnitudes of its terms
  (the bound the tensor-core convolution tests use), propagated through |W| (ReLU is 1-Lipschitz) to per-row error norms e_f, e_t;
  a score moves by <= e_f + e_t (triangle inequality), a log-softmax by that plus the largest such move, and the host's fp32
  prior by u |prior|.  That bound is dominated by the convolutions' 2^-14: the measured error is 1.4e-5 of it at adim 128,
  9.2e-6 at 256 and 7.4e-6 at 512 (the distance / log-softmax stage itself is held to tau above).

* get_segments copies: bit for bit.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from emotivoice_b200 import align, feats, synth
from oracle import align_oracle as AO

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
MAS_FIXTURES = ["mas_t255", "mas_t256", "mas_t257", "mas_t513", "mas_b16", "mas_edges", "mas_ties", "mas_ninf"]
AVG_FIXTURES = ["avg_energy", "avg_logpitch"]


def _np(name):
    return {k: v.numpy() for k, v in load_golden(name).items()}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _i64(v):
    return torch.as_tensor(np.asarray(v), dtype=torch.int64).to(DEV)


def mas(lib, lp, tl, fl):
    """ev_op_mas on (B, F, T) float32 -> (path, durations, per-item loss) on the host; outputs start as sentinels."""
    B, Fp, T = lp.shape
    lp_d = torch.as_tensor(lp).to(DEV).contiguous()
    path = torch.full((B, Fp), -7, dtype=torch.int32, device=DEV)
    ds = torch.full((B, T), -7.0, device=DEV)
    loss = torch.full((B,), -7.0, device=DEV)
    ws = torch.empty(B * Fp * T, dtype=torch.uint8, device=DEV)
    tl_d, fl_d = _i64(tl), _i64(fl)
    rc = lib.ev_op_mas(lp_d.data_ptr(), tl_d.data_ptr(), fl_d.data_ptr(), B, Fp, T, path.data_ptr(), ds.data_ptr(), loss.data_ptr(),
                       ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    return rc, path.cpu().numpy(), ds.cpu().numpy(), loss.cpu().numpy()


def avg(lib, d, xs, tl, fl):
    B, T = d.shape
    d_d, x_d = torch.as_tensor(d).to(DEV).contiguous(), torch.as_tensor(xs).to(DEV).contiguous()
    out = torch.full((B, T), -7.0, device=DEV)
    tl_d, fl_d = _i64(tl), _i64(fl)
    rc = lib.ev_op_average_by_duration(d_d.data_ptr(), x_d.data_ptr(), tl_d.data_ptr(), fl_d.data_ptr(), B, x_d.shape[1], T, out.data_ptr(), _st())
    torch.cuda.synchronize()
    return rc, out.cpu().numpy()


def logp(lib, text, fts, tl, prior):
    B, T, A = text.shape
    out = torch.full((B, fts.shape[1], T), -7.0, device=DEV)
    tl_d = None if tl is None else _i64(tl)
    rc = lib.ev_op_align_logp(text.data_ptr(), fts.data_ptr(), None if tl_d is None else tl_d.data_ptr(), None if prior is None else prior.data_ptr(),
                              B, fts.shape[1], T, A, out.data_ptr(), _st())
    torch.cuda.synchronize()
    return rc, out


def check_loss(loss, lp, path, fl):
    for b, f in enumerate(fl):
        if f <= 0:
            continue
        m64 = -np.float64(lp[b, np.arange(f), path[b, :f]].astype(np.float64).mean())
        want = np.float32(m64)
        if not np.isfinite(want):
            assert loss[b] == want, (b, loss[b], want)
        else:
            assert abs(np.float64(loss[b]) - np.float64(want)) <= np.spacing(np.abs(want)), (b, loss[b], want)


# ---- monotonic alignment search -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", MAS_FIXTURES + ["mas_row0"])
def test_mas_equals_reference_at_training_shapes(lib, name):
    """Paths and durations identical to the reference's numba search (T_inp 255/256/257/513, F up to 1800, B = 16, F < T_inp,
    F == T_inp, F == 1, T == 1, ties, -inf cells, the crafted row-0 case); per-item losses within 1 ulp of fl32(-mean64)."""
    g = _np(name)
    lp = g["log_p_attn"] if name == "mas_row0" else AO.band_log_p(g["text_lengths"], g["feats_lengths"], int(g["T_pad"]), int(g["F_pad"]),
                                                                  int(g["seed"]), AO.MAS_KINDS[int(g["kind"])])
    tl, fl = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    rc, path, ds, loss = mas(lib, lp, tl, fl)
    assert rc == 0
    assert np.array_equal(path, g["paths"].astype(np.int32))
    if "durations" in g:
        assert np.array_equal(ds, g["durations"].astype(np.float32))
        assert all(a == b or abs(float(a) - float(b)) <= 1e-6 * abs(float(b)) for a, b in zip(loss, g["item_bin_loss"]))
    else:
        assert not np.array_equal(path, g["float64_row0_path"].astype(np.int32))
    check_loss(loss, lp, path, fl)


def test_mas_equals_oracle_on_random_log_softmax(lib):
    """Generated log-softmax rows (the shape AlignmentModule produces) at B = 8, T_inp 300, F up to 1500, vs the oracle."""
    g = torch.Generator().manual_seed(31)
    tl, fl = [300, 257, 1, 64, 180, 299, 12, 256], [1500, 1100, 40, 64, 30, 900, 12, 1]
    score = torch.randn(8, 1500, 300, generator=g) * 2.0
    for b in range(8):
        score[b, :, tl[b]:] = -np.inf
    lp = torch.log_softmax(score, dim=-1).numpy()
    rc, path, ds, loss = mas(lib, lp, tl, fl)
    assert rc == 0
    o_ds, _ = AO.viterbi_decode(lp, tl, fl)
    assert np.array_equal(ds, o_ds)
    for b in range(8):
        assert np.array_equal(path[b, :fl[b]], AO.monotonic_alignment_search(lp[b, :fl[b], :tl[b]])) and (path[b, fl[b]:] == -1).all()
    check_loss(loss, lp, path, fl)


def test_mas_items_are_independent_of_the_batch(lib):
    """Each item of a ragged batch equals its own B=1 call bit for bit; NaN outside each item's rectangle changes nothing;
    lengths above the padded sizes act as the padded sizes."""
    g = _np("mas_b16")
    tl, fl = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    lp = AO.band_log_p(tl, fl, int(g["T_pad"]), int(g["F_pad"]), int(g["seed"]), "band")
    rc, path, ds, loss = mas(lib, lp, tl, fl)
    assert rc == 0
    poisoned = lp.copy()
    for b in range(len(tl)):
        poisoned[b, fl[b]:, :] = np.nan
        poisoned[b, :, tl[b]:] = np.nan
    rc, p2, d2, l2 = mas(lib, poisoned, tl, fl)
    assert rc == 0 and np.array_equal(p2, path) and np.array_equal(d2, ds) and np.array_equal(l2, loss)
    for b in (0, 3, 7, 15):
        rc, p1, d1, l1 = mas(lib, np.ascontiguousarray(lp[b:b + 1, :fl[b], :tl[b]]), [tl[b]], [fl[b]])
        assert rc == 0 and np.array_equal(p1[0], path[b, :fl[b]]) and np.array_equal(d1[0], ds[b, :tl[b]]) and l1[0] == loss[b]
        assert (ds[b, tl[b]:] == 0).all()
    T_pad, F_pad = lp.shape[2], lp.shape[1]
    big = np.ascontiguousarray(lp[3:4])                                 # item 3 fills the padded frames (F = 1800)
    rc, p_at, d_at, l_at = mas(lib, big, [T_pad], [F_pad])
    rc2, p_over, d_over, l_over = mas(lib, big, [T_pad + 5], [F_pad + 7])
    assert rc == 0 and rc2 == 0 and np.array_equal(p_at, p_over) and np.array_equal(d_at, d_over) and np.array_equal(l_at, l_over)


def test_mas_shared_memory_cap(lib):
    """T_inp = 10240 tokens (the 200 KB shared-memory budget) runs and matches the oracle; 10241 is refused before any launch:
    the outputs keep their sentinels."""
    tl, fl = [10240], [12]
    lp = AO.band_log_p(tl, fl, 10240, 12, 7301, "band")
    rc, path, ds, loss = mas(lib, lp, tl, fl)
    assert rc == 0
    assert np.array_equal(path[0], AO.monotonic_alignment_search(lp[0]))
    assert np.array_equal(ds, AO.viterbi_decode(lp, tl, fl)[0])
    check_loss(loss, lp, path, fl)
    lp2 = np.zeros((1, 12, 10241), np.float32)
    rc, path, ds, loss = mas(lib, lp2, [10241], [12])
    assert rc != 0
    assert (path == -7).all() and (ds == -7).all() and (loss == -7).all()


# ---- per-token averaging --------------------------------------------------------------------------------------------------

def avg_bound(d, xs, tl, fl):
    """1 ulp of fl32(mean64) plus the float64 sum's n 2^-53 mean|x|, per element; and mean64 itself."""
    m64 = AO.average_by_duration64(d, xs, tl, fl)
    mabs = AO.average_by_duration64(d, np.abs(xs), tl, fl)
    n = np.zeros_like(m64)
    for b, k, seg in AO._token_slices(d, xs, tl, fl):
        n[b, k] = len(seg)
    ulp = np.spacing(np.abs(m64).astype(np.float32)).astype(np.float64)
    ulp[n == 0] = 0.0
    return m64, ulp + n * 2.0 ** -53 * mabs


def check_avg(y, d, xs, tl, fl, what):
    m64, bnd = avg_bound(d, xs, tl, fl)
    err = np.abs(y.astype(np.float64) - m64.astype(np.float32).astype(np.float64))
    assert (err <= bnd).all(), (what, np.argwhere(err > bnd)[:5], err.max())
    nz = bnd > 0
    print("%s: largest |y - fl32(mean64)| = %.2f ulp" % (what, (err[nz] / bnd[nz]).max() if nz.any() else 0.0))
    return m64


@pytest.mark.parametrize("name", AVG_FIXTURES)
def test_average_by_duration_at_track_magnitudes(lib, name):
    """Energy- and log-pitch-like tracks: within 1 ulp of fl32(mean64) everywhere, within that plus the stored deviation of the
    reference; zeros past text_lens; NaN past feats_lens is not read; T_inp > 256; lengths past the padded sizes."""
    g = _np(name)
    d = g["durations"].astype(np.float32)
    xs = g["xs_q"].astype(np.float32) * np.float32(2.0 ** -int(g["xs_log2_scale"]))
    tl, fl = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    rc, y = avg(lib, d, xs, tl, fl)
    assert rc == 0
    m64, bnd = avg_bound(d, xs, tl, fl)
    check_avg(y, d, xs, tl, fl, name)
    assert (np.abs(y.astype(np.float64) - g["averaged"].astype(np.float64)) <= bnd + g["averaged_dev"]).all()
    for b, t in enumerate(tl):
        assert (y[b, t:] == 0).all()
    poisoned = xs.copy()
    for b, f in enumerate(fl):
        poisoned[b, f:] = np.nan
    rc, y2 = avg(lib, d, poisoned, tl, fl)
    assert rc == 0 and np.array_equal(y2, y) and np.isfinite(y2).all()
    if name == "avg_energy":
        assert d.shape[1] > 256 and max(tl) > d.shape[1] and max(fl) > xs.shape[1]


def test_average_by_duration_negative_durations_stay_inside_the_item(lib):
    """Negative durations slice the item's row the way numpy does (the reference's semantics).  The item sits at b = 1 between
    rows of NaN: a bound that left [0, F) would read them (a NaN or a wrong finite value), never memory outside the tensor."""
    Fp, T = 40, 9
    rng = np.random.default_rng(17)
    xs = np.full((3, Fp), np.nan, np.float32)
    xs[1] = (rng.integers(5 << 17, 100 << 17, Fp) * 2.0 ** -17).astype(np.float32)
    d = np.zeros((3, T), np.float32)
    d[1] = [-2, 5, 4, -3, 7, 0, -1, 30, 6]                             # cumsum -2 3 7 4 11 11 10 40 46: x[0:-2], x[-2:3], ...
    tl, fl = [0, T, 0], [0, 35, 0]
    rc, y = avg(lib, d, xs, tl, fl)
    assert rc == 0
    want = AO.average_by_duration(d, xs, tl, fl)                       # bit for bit the reference's numba loop
    assert np.isfinite(y).all(), y[1]
    m64, bnd = avg_bound(d, xs, tl, fl)
    check_avg(y, d, xs, tl, fl, "negative durations")
    assert (np.abs(y.astype(np.float64) - want.astype(np.float64)) <= bnd + np.abs(want.astype(np.float64) - m64)).all()
    assert y[1, 0] != 0 and y[1, 1] == 0 and (y[0] == 0).all() and (y[2] == 0).all()
    assert abs(m64[1, 0] - np.mean(xs[1, :33].astype(np.float64))) <= 1e-12 * m64[1, 0]      # x[0:-2] of the 35-frame item


def test_energy_and_pitch_token_averages_are_fp64_means(lib):
    """feats.Energy.get_energy(duration=) and feats.Pitch.get_pitch(use_token_averaged_pitch=True, duration=) against the
    float64 mean of their own frame tracks (the track rounded to float32 adds <= u max|x| over the token)."""
    sr = 24000
    t = np.arange(2 * sr) / sr
    wav = (0.3 * np.sin(2 * np.pi * 180 * t * (1 + 0.1 * t)) + 0.01 * np.random.default_rng(3).normal(size=t.size)).astype(np.float32)
    w = torch.from_numpy(wav).to(DEV)
    en = feats.Energy(sr=sr, n_fft=1024, hop_length=256, win_length=1024)
    pt = feats.Pitch(sr=sr, hop_length=300)
    for name, track, tok in (("energy", lambda: en.get_energy(w, use_token_averaged_energy=False), lambda d: en.get_energy(w, duration=d)),
                             ("pitch", lambda: pt.get_pitch(w), lambda d: pt.get_pitch(w, use_token_averaged_pitch=True, duration=d))):
        x = track().double().cpu().numpy()[None]
        Fn = x.shape[1]
        d = np.array([3, 0, 11, 25, 1, 7, 40, 13, 0, 9, 30, 60], np.float32)      # sums past the track's frames
        y = tok(torch.from_numpy(d)).double().cpu().numpy()[None]
        m64 = AO.average_by_duration64(d[None], x, [d.size], [Fn])
        bnd = np.spacing(np.abs(m64).astype(np.float32)).astype(np.float64) + U * np.abs(x).max()
        bnd[m64 == 0] = 0.0
        assert (np.abs(y - m64) <= bnd).all(), (name, np.abs(y - m64).max())


# ---- distance / log-softmax ----------------------------------------------------------------------------------------------

def logp_bound(NC, tl):
    c_s = NC / 2 + 6
    tau = (3 * c_s + 4) * U
    kappa = ((4 * c_s + 5) * math.log(max(tl, 1)) + math.ceil(tl / 32) + 9) * U
    return tau, kappa


def check_logp(out, lp64, s_abs, l_abs, tls, NC, what):
    """The -inf pattern identical, finite entries within the derived bound.  Returns the largest err / (|s| + |lse|)."""
    out = out.double()
    fin = torch.isfinite(lp64)
    assert torch.equal(fin, torch.isfinite(out)), what
    assert (out[~fin] == -np.inf).all() and (lp64[~fin] == -np.inf).all(), what
    worst = 0.0
    for b, tl in enumerate(tls):
        tau, kappa = logp_bound(NC, tl)
        f = fin[b]
        m = (s_abs[b] + l_abs[b])[f]
        err = (out[b] - lp64[b])[f].abs()
        bnd = tau * m + kappa + U * lp64[b][f].abs()
        assert (err <= bnd).all(), (what, b, (err / bnd).max().item())
        if err.numel():
            worst = max(worst, (err / m.clamp_min(1e-30)).max().item())
    return worst


@pytest.mark.parametrize("A", [128, 256, 384, 512])
def test_align_logp_against_fp64(lib, A):
    """T in {1, 31, 32, 33, 3072}, F in {1, 2, 3, 5, 1201}; text_lens 1, T and > T in one batch (text rows past them NaN) with a
    prior, and text_lens null without one.  Each item equals its own B=1 call bit for bit; T = 3073 is refused before launch."""
    NC = A // 128
    g = torch.Generator(device=DEV).manual_seed(A)
    worst = 0.0
    for T in (1, 31, 32, 33, 3072):
        for Fn in (1, 2, 3, 5, 1201):
            text = torch.randn(3, T, A, generator=g, device=DEV)
            fts = torch.randn(3, Fn, A, generator=g, device=DEV) * 1.2
            tls = [T, 1, T + 7]
            eff = [min(v, T) for v in tls]
            poisoned = text.clone()
            for b, v in enumerate(eff):
                poisoned[b, v:] = np.nan
            prior = torch.randn(3, Fn, T, generator=g, device=DEV) * 3.0 - 2.0
            prior[1, :, 1:] = -np.inf                                  # -inf outside item 1's rectangle, as the real prior has
            prior[2, Fn // 2 + 1:, :] = -np.inf
            rc, out = logp(lib, poisoned, fts, tls, prior)
            assert rc == 0
            lp64, s_abs, l_abs = AO.align_logp64(text, fts, torch.tensor(tls), prior)
            worst = max(worst, check_logp(out, lp64, s_abs, l_abs, eff, NC, (A, T, Fn, "lens+prior")))
            for b in range(3):
                rc, one = logp(lib, poisoned[b:b + 1].contiguous(), fts[b:b + 1].contiguous(), tls[b:b + 1], prior[b:b + 1].contiguous())
                assert rc == 0 and torch.equal(one[0], out[b]), (A, T, Fn, b)
            rc, out = logp(lib, text, fts, None, None)
            assert rc == 0
            lp64, s_abs, l_abs = AO.align_logp64(text, fts)
            worst = max(worst, check_logp(out, lp64, s_abs, l_abs, [T] * 3, NC, (A, T, Fn, "null")))
    tau, _ = logp_bound(NC, 3072)
    print("align_logp A=%d: largest err/(|s|+|lse|) = 2^%.1f (tau 2^%.1f)" % (A, math.log2(max(worst, 1e-300)), math.log2(tau)))
    text = torch.zeros(1, 3073, A, device=DEV)
    fts = torch.zeros(1, 2, A, device=DEV)
    rc, out = logp(lib, text, fts, None, None)
    assert rc != 0 and (out == -7).all()


def _conv_chain(sd, x, names, adim):
    """The module's convolution chain in float64 with the error each 3xTF32 layer may add (2^-14 of the magnitudes of its
    terms), propagated through |W|.  Returns (output, per-element error bound)."""
    h, e = x, torch.zeros_like(x)
    for name, k, relu in names:
        w, bias = sd[name + ".weight"].double().to(DEV), sd[name + ".bias"].double().to(DEV)
        pad = (k - 1) // 2
        y = F.conv1d(h.transpose(1, 2), w, bias, padding=pad).transpose(1, 2)
        mag = F.conv1d(h.abs().transpose(1, 2), w.abs(), bias.abs(), padding=pad).transpose(1, 2)
        e = F.conv1d(e.transpose(1, 2), w.abs(), None, padding=pad).transpose(1, 2) + 2.0 ** -14 * mag
        h = F.relu(y) if relu else y
    return h, e


@pytest.mark.parametrize("adim", [128, 256, 512])
def test_alignment_module_other_widths_against_fp64(lib, adim):
    """AlignmentModule at adim 128, 256 and 512 against the oracle's forward in float64 (the -inf pattern identical)."""
    odim = 80
    sd = synth.make_alignment_state_dict(adim, odim)
    mod = align.AlignmentModule(adim, odim).to(DEV)
    mod.load_state_dict(sd)
    tl, fl = torch.tensor([23, 9, 31]), torch.tensor([120, 40, 187])
    B, T, Fn = 3, 31, 187
    rng = np.random.default_rng(8000 + adim)
    text = torch.from_numpy(rng.normal(size=(B, T, adim)).astype(np.float32)).to(DEV)
    fts = torch.from_numpy((rng.normal(size=(B, Fn, odim)) * 1.2).astype(np.float32)).to(DEV)
    x_masks = (torch.arange(T)[None, :] >= tl[:, None]).to(DEV)
    out = mod(text, fts, tl, fl, x_masks).double()
    prior64 = mod._generate_prior(tl, fl).double().to(DEV)
    sd64 = {k: v.double().to(DEV) for k, v in sd.items()}
    ref = AO.alignment_module_forward(sd64, text.double(), fts.double(), tl, fl, x_masks, prior_fn=lambda a, b: prior64)
    t64, et = _conv_chain(sd, text.double(), (("t_conv1", 3, True), ("t_conv2", 1, False)), adim)
    f64, ef = _conv_chain(sd, fts.double(), (("f_conv1", 3, True), ("f_conv2", 3, True), ("f_conv3", 1, False)), adim)
    lp64, s_abs, l_abs = AO.align_logp64(t64, f64, tl, prior64)
    fin = torch.isfinite(ref)
    assert torch.equal(fin, torch.isfinite(lp64)) and (ref - lp64)[fin].abs().max() <= 1e-9
    assert torch.equal(fin, torch.isfinite(out))
    e_t, e_f = et.norm(dim=-1), ef.norm(dim=-1)                         # (B, T), (B, F)
    worst = 0.0
    for b in range(B):
        n = int(tl[b])
        tau, kappa = logp_bound(adim // 128, n)
        ds = e_f[b][:, None] + e_t[b][None, :n]                         # |score error| from the convolutions
        bnd = ds + ds.max(dim=1, keepdim=True).values + tau * (s_abs[b, :, :n] + l_abs[b]) + kappa + U * lp64[b, :, :n].abs() + U * prior64[b, :, :n].abs()
        f = fin[b, :, :n]
        err = (out[b, :, :n] - ref[b, :, :n]).abs()
        assert (err[f] <= bnd[f]).all(), (adim, b, (err[f] / bnd[f]).max().item())
        worst = max(worst, (err[f] / bnd[f]).max().item())
    print("AlignmentModule adim=%d: largest err / bound = %.3g" % (adim, worst))


# ---- segments ------------------------------------------------------------------------------------------------------------

def test_get_segments_bit_exact_at_the_edges(lib):
    """out[b, :, i] = x[b, :, start + i] while start + i < T, else 0: start + seg > T, seg > T, T = 1."""
    g = torch.Generator().manual_seed(11)
    for B, C, T, seg, starts in ((3, 80, 50, 32, [0, 18, 49]), (2, 7, 20, 64, [0, 5]), (2, 3, 1, 5, [0, 0]), (4, 192, 300, 256, [44, 0, 299, 12])):
        x = torch.randn(B, C, T, generator=g)
        st = torch.tensor(starts)
        want = torch.zeros(B, C, seg)
        for b in range(B):
            s = starts[b]
            n = max(0, min(seg, T - s))
            want[b, :, :n] = x[b, :, s:s + n]
        got = align.get_segments(x.to(DEV), st.to(DEV), seg).cpu()
        assert torch.equal(got, want), (B, C, T, seg)
