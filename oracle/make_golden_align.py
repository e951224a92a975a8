"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/align_*.npz, mas_*.npz and avg_*.npz from the reference's own numba functions
(models/prompt_tts_modified/modules/alignment.py:90-177: _monotonic_alignment_search via viterbi_decode, average_by_duration)
and pins oracle/align_oracle.py against them.  Run in the build container:  python oracle/make_golden_align.py
Inputs are log-softmax rows like AlignmentModule.forward produces (alignment.py:47) -- one case quantised so that ties between
the two predecessor cells are frequent (the tie rule decides the integer path)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import align_oracle as AO      # noqa: E402
from oracle import refshim                 # noqa: E402

CASES = {
    # name: (text lengths, feats lengths, seed, quantise)
    "align_b3": ([17, 9, 25], [80, 33, 140], 7001, False),
    "align_b2_ties": ([12, 30], [64, 200], 7002, True),
    "align_b4_long": ([100, 57, 3, 120], [537, 260, 3, 600], 7003, False),     # incl. T_mel == T_inp and the bench utterance's shape
}


def main():
    if refshim.REF_ROOT not in sys.path:
        sys.path.insert(0, refshim.REF_ROOT)
    from models.prompt_tts_modified.modules import alignment as R
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, (tt, tf, seed, quant) in CASES.items():
        rng = np.random.default_rng(seed)
        B, T, F = len(tt), max(tt), max(tf)
        score = rng.normal(size=(B, F, T)).astype(np.float32) * 2.0
        for b in range(B):
            score[b, :, tt[b]:] = -np.inf                                  # x_masks (alignment.py:43-45)
        lp = torch.log_softmax(torch.from_numpy(score), dim=-1)
        if quant:
            lp = torch.round(lp * 4) / 4
        tl, fl = torch.tensor(tt), torch.tensor(tf)
        ds, bin_loss = R.viterbi_decode(lp, tl, fl)
        xs = torch.from_numpy(rng.normal(size=(B, F)).astype(np.float32))
        avg = R.average_by_duration(ds, xs, tl, fl)
        paths = np.full((B, F), -1, np.int32)
        for b in range(B):
            paths[b, :tf[b]] = R._monotonic_alignment_search(lp[b, :tf[b], :tt[b]].numpy())
        o_ds, o_bl = AO.viterbi_decode(lp.numpy(), tt, tf)
        o_avg = AO.average_by_duration(o_ds, xs.numpy(), tt, tf)
        assert np.array_equal(o_ds, ds.numpy()) and abs(float(o_bl) - float(bin_loss)) <= 1e-6 * abs(float(bin_loss)), name
        assert np.array_equal(o_avg, avg.numpy()), name
        for b in range(B):
            assert np.array_equal(AO.monotonic_alignment_search(lp[b, :tf[b], :tt[b]].numpy()), paths[b, :tf[b]]), name
        _save(name, log_p_attn=lp.numpy(), text_lengths=np.asarray(tt, np.int64), feats_lengths=np.asarray(tf, np.int64), xs=xs.numpy(),
              paths=paths, durations=ds.numpy(), bin_loss=np.float32(bin_loss), averaged=avg.numpy())
        print(name, "ok: bin_loss %.6f, durations sum %s" % (float(bin_loss), ds.sum(1).tolist()))


def _save(name, **arrays):
    """Writes tests/golden/<name>.npz unless a file with exactly these arrays is already there (keeps regeneration a no-op)."""
    path = os.path.join(ROOT, "tests", "golden", name + ".npz")
    if os.path.exists(path):
        with np.load(path) as z:
            if sorted(z.files) == sorted(arrays) and all(z[k].dtype == np.asarray(v).dtype and np.array_equal(z[k], v, equal_nan=True)
                                                        for k, v in arrays.items()):
                return
    np.savez_compressed(path, **arrays)


def _reference():
    if refshim.REF_ROOT not in sys.path:
        sys.path.insert(0, refshim.REF_ROOT)
    from models.prompt_tts_modified.modules import alignment as R
    return R


# Monotonic alignment search at training shapes and edges.  The inputs are not stored: AO.band_log_p rebuilds them bit for bit
# from (lengths, padded sizes, seed, kind); the fixture keeps the reference's paths, durations and per-item bin losses.
MAS_CASES = {
    # name: (text lengths, feats lengths, T_pad, F_pad, seed, kind)
    "mas_t255": ([255, 200, 100, 37], [1200, 900, 500, 150], 255, 1200, 7101, "band"),
    "mas_t256": ([256, 256, 9], [1100, 256, 40], 256, 1100, 7102, "band"),                     # F == T_inp in item 1
    "mas_t257": ([257, 130, 257], [1800, 700, 300], 257, 1800, 7103, "band"),                  # threads stride over tokens
    "mas_t513": ([513, 400], [1700, 1500], 513, 1700, 7104, "band"),
    "mas_b16": ([61, 143, 97, 180, 12, 77, 150, 33, 120, 88, 170, 45, 101, 66, 129, 20],
                [390, 1010, 600, 1800, 70, 455, 1200, 160, 790, 610, 1400, 300, 720, 380, 900, 95], 180, 1800, 7105, "band"),
    "mas_edges": ([40, 60, 5, 1, 1, 2], [25, 60, 1, 90, 1, 2], 60, 90, 7106, "band"),           # F < T, F == T, F == 1, T == 1, both 1
    "mas_ties": ([30, 75, 128], [120, 300, 640], 128, 640, 7107, "ties"),
    "mas_ninf": ([40, 90, 260], [200, 410, 1000], 260, 1000, 7108, "ninf"),                     # -inf cells inside the rectangles
}


def make_mas_fixtures():
    import torch
    R = _reference()
    for name, (tt, tf, T_pad, F_pad, seed, kind) in MAS_CASES.items():
        lp = AO.band_log_p(tt, tf, T_pad, F_pad, seed, kind)
        B = len(tt)
        paths = np.full((B, F_pad), -1, np.int16)
        losses = np.zeros(B, np.float32)
        for b in range(B):
            cur = lp[b, :tf[b], :tt[b]]
            p = R._monotonic_alignment_search(cur)
            paths[b, :tf[b]] = p
            losses[b] = -torch.from_numpy(cur)[torch.arange(tf[b]), torch.from_numpy(p)].mean().item()     # viterbi_decode's per-item term
            assert np.array_equal(AO.monotonic_alignment_search(cur), p), (name, b)
        ds, bin_loss = R.viterbi_decode(torch.from_numpy(lp), torch.tensor(tt), torch.tensor(tf))
        assert np.array_equal(AO.viterbi_decode(lp, tt, tf)[0], ds.numpy()), name
        _save(name, text_lengths=np.asarray(tt, np.int64), feats_lengths=np.asarray(tf, np.int64), T_pad=np.int64(T_pad), F_pad=np.int64(F_pad),
              seed=np.int64(seed), kind=np.int64(AO.MAS_KINDS.index(kind)), paths=paths, durations=ds.numpy().astype(np.int16),
              item_bin_loss=losses, bin_loss=np.float32(bin_loss))
        print(name, "ok: durations sum", ds.sum(1).int().tolist())


def _row0_alternatives(lp):
    """The path the search would take with row 0 summed in float64, and summed pairwise in float32 (numpy's sum)."""
    out = []
    for row0 in (lambda r: np.cumsum(r.astype(np.float64)),
                 lambda r: np.array([np.sum(r[:j + 1], dtype=np.float32) for j in range(len(r))], np.float64)):
        T_inp, T_mel = lp.shape[1], lp.shape[0]
        Q = np.full((T_inp, T_mel), -np.inf)
        Q[0] = row0(lp[:, 0])
        for j in range(1, T_mel):
            for i in range(1, min(j + 1, T_inp)):
                Q[i, j] = max(Q[i - 1, j - 1], Q[i, j - 1]) + np.float64(lp[j, i])
        A = np.full((T_mel,), T_inp - 1)
        for j in range(T_mel - 2, -1, -1):
            A[j] = 0 if A[j + 1] == 0 else (A[j + 1] - 1 if Q[A[j + 1] - 1, j] >= Q[A[j + 1], j] else A[j + 1])
        out.append(A)
    return out


def make_row0_fixture():
    """A search decided by the last bit of row 0, which the reference sums sequentially in float32.  Token 1 costs -1000 before
    frame j*, 0 after it, and at j* its score is c = the score of token 0 at j*.  The backtrack stays on token 1 down to j*
    (token 0's running sum only falls), and there it compares
    fl32(S + c) >= S + c, S = the float32 running sum of token 0 over frames < j*.  The inputs are chosen so that fl32 rounds
    down: the reference then keeps token 1 at j*, while a float64 row 0 would tie and (ties -> token 0) not."""
    R = _reference()
    rng = np.random.default_rng(7109)
    jstar, F, T = 57, 60, 2
    while True:
        lp = np.full((F, T), -1000.0, np.float32)
        lp[:, 0] = -rng.uniform(0.01, 3.0, F).astype(np.float32)
        S = np.cumsum(lp[:jstar, 0], dtype=np.float32)[-1]
        c = lp[jstar, 0]
        lp[jstar, 1] = c
        lp[jstar + 1:, 1] = 0.0
        if np.float64(np.float32(S + c)) < np.float64(S) + np.float64(c) and np.float64(S) != np.cumsum(lp[:jstar, 0].astype(np.float64))[-1]:
            break
    p = R._monotonic_alignment_search(lp)
    assert np.array_equal(AO.monotonic_alignment_search(lp), p)
    alt64, alt_pw = _row0_alternatives(lp)
    assert not np.array_equal(alt64, p), "a float64 row 0 must give a different path, or this case does not pin row 0"
    print("mas_row0 ok: reference keeps token 1 from frame %d; float64 row 0 from frame %d; pairwise row 0 %s" % (
        int(np.argmax(p)), int(np.argmax(alt64)), "differs" if not np.array_equal(alt_pw, p) else "agrees"))
    _save("mas_row0", log_p_attn=lp[None], text_lengths=np.array([T], np.int64), feats_lengths=np.array([F], np.int64),
          paths=p.astype(np.int16)[None], float64_row0_path=alt64.astype(np.int16)[None])


# Per-token averaging at the magnitudes of the tracks it averages.  Each track is an integer below 2^24 times a power of two, so
# exact in float32 and stored exactly (int32), with the low bits random so that the reference's float32 running sums round.
def _avg_case(seed, B, F_pad, T_pad, lo, hi, shift, items):
    """items: per item (text length, feats length, duration recipe).  Returns (xs_q int32, durations int16, lengths)."""
    rng = np.random.default_rng(seed)
    xs_q = np.zeros((B, F_pad), np.int32)
    for b in range(B):                                                  # a random walk between lo and hi (in units of 2^-shift)
        w = np.cumsum(rng.integers(-40 << (shift - 8), 41 << (shift - 8), F_pad)) + rng.integers(lo, hi)
        w = np.abs((w - lo) % (2 * (hi - lo)) - (hi - lo)) + lo
        xs_q[b] = w.astype(np.int32)
    ds = np.zeros((B, T_pad), np.int16)
    tl, fl = [], []
    for b, (t, f, kind) in enumerate(items):
        n = min(t, T_pad)
        if kind == "short":                                             # 1-30 frames, some zero
            d = rng.integers(0, 31, n)
        elif kind == "long":                                            # a few very long tokens among short ones
            d = rng.integers(1, 12, n)
            d[rng.integers(0, n, 3)] = rng.integers(150, 600, 3)
        elif kind == "negative":                                        # negative durations: numpy slice semantics decide
            d = rng.integers(-6, 25, n)
            d[:3] = [-3, 2, 8]                                          # bounds -3, -1, 7: x[0:-3], x[-3:-1], x[-1:7]
        else:                                                           # "exact": sum == the feats length
            d = rng.multinomial(f, np.ones(n) / n)
        ds[b, :n] = d
        tl.append(t)
        fl.append(f)
    return xs_q, ds, tl, fl


AVG_CASES = {
    # name: (seed, T_pad, F_pad, lo, hi, log2 scale, items (text length, feats length, durations))
    "avg_energy": (7201, 300, 1800, 5 << 17, 100 << 17, 17,
                   [(120, 1800, "short"), (300, 1800, "short"), (80, 1500, "long"), (40, 900, "exact"), (60, 700, "negative"),
                    (200, 1800, "negative"), (310, 1900, "short"), (1, 1, "exact")]),
    "avg_logpitch": (7202, 260, 1200, int(4.38 * 2 ** 21), int(5.99 * 2 ** 21), 21,
                     [(90, 1200, "short"), (260, 1200, "long"), (50, 400, "negative"), (30, 1200, "exact"), (100, 300, "short")]),
}


def make_avg_fixtures():
    import torch
    R = _reference()
    for name, (seed, T_pad, F_pad, lo, hi, shift, items) in AVG_CASES.items():
        B = len(items)
        xs_q, ds, tl, fl = _avg_case(seed, B, F_pad, T_pad, lo, hi, shift, items)
        xs = xs_q.astype(np.float32) * np.float32(2.0 ** -shift)
        d = ds.astype(np.float32)
        ref = R.average_by_duration(torch.from_numpy(d), torch.from_numpy(xs), torch.tensor(tl), torch.tensor(fl)).numpy()
        o = AO.average_by_duration(d, xs, tl, fl)
        assert np.array_equal(o, ref), name                             # the oracle restates the reference bit for bit
        m64 = AO.average_by_duration64(d, xs, tl, fl)
        dev = np.abs(ref.astype(np.float64) - m64)
        nz = m64 != 0
        print("%s ok: reference vs float64 mean: max %.3g (%.2f ulp), %d of %d differ from fl32(mean64)" % (
            name, dev.max(), (dev[nz] / np.spacing(np.abs(m64[nz]).astype(np.float32))).max(), int((ref != m64.astype(np.float32)).sum()), int(nz.sum())))
        _save(name, xs_q=xs_q, xs_log2_scale=np.int64(shift), durations=ds, text_lengths=np.asarray(tl, np.int64),
              feats_lengths=np.asarray(fl, np.int64), averaged=ref, averaged_dev=dev)


def make_module_fixture():
    """AlignmentModule.forward + get_random_segments of the UNMODIFIED reference on seeded inputs -> tests/golden/alignmod_b3.npz."""
    if refshim.REF_ROOT not in sys.path:
        sys.path.insert(0, refshim.REF_ROOT)
    from models.prompt_tts_modified.modules import alignment as R
    from models.hifigan import get_random_segments as RS
    from emotivoice_b200 import synth
    adim, odim = 384, 80
    mod = R.AlignmentModule(adim, odim).eval()
    mod.load_state_dict(synth.make_alignment_state_dict(adim, odim), strict=True)       # seeded: the fixture need not carry the weights
    tt, tf = [23, 9, 31], [120, 40, 187]
    B, T, F = len(tt), max(tt), max(tf)
    rng = np.random.default_rng(8001)
    text = torch.from_numpy(rng.normal(size=(B, T, adim)).astype(np.float32))
    feats = torch.from_numpy((rng.normal(size=(B, F, odim)) * 1.2).astype(np.float32))
    tl, fl = torch.tensor(tt), torch.tensor(tf)
    x_masks = torch.arange(T)[None, :] >= tl[:, None]                         # True = pad (model_open_source.py:164-173)
    with torch.no_grad():
        lp = mod(text, feats, tl, fl, x_masks)
    sd = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    o = AO.alignment_module_forward(sd, text, feats, tl, fl, x_masks, prior_fn=mod._generate_prior)
    fin = torch.isfinite(lp)
    assert torch.equal(fin, torch.isfinite(o)) and (lp[fin] - o[fin]).abs().max() <= 1e-5, "oracle restatement differs from the reference module"
    torch.manual_seed(99)
    z = torch.from_numpy(rng.normal(size=(B, odim, F)).astype(np.float32))
    seg, starts, size = RS.get_random_segments(z, fl, 32)
    assert np.array_equal(AO.get_segments(z.numpy(), starts.numpy(), 32), seg.numpy())
    short = RS.get_segments(z[:, :, :20], torch.tensor([0, 3, 19]), 32)        # t < segment_size: zero padded
    arrays = {"text": text.numpy(), "feats": feats.numpy(), "text_lengths": tl.numpy().astype(np.int64), "feats_lengths": fl.numpy().astype(np.int64),
              "log_p_attn": lp.numpy(), "z": z.numpy(), "seg": seg.numpy(), "starts": starts.numpy().astype(np.int64), "seg_short": short.numpy()}
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "alignmod_b3.npz"), **arrays)
    print("alignmod_b3 ok: log_p_attn", tuple(lp.shape), "starts", starts.tolist())


if __name__ == "__main__":
    main()
    make_module_fixture()
    make_mas_fixtures()
    make_row0_fixture()
    make_avg_fixtures()
