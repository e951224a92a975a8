"""The true-peak limiter on the GPU (``format_audio(true_peak=...)``, ev_limit): the envelope and samples against the fp64
oracle on synthetic items and the engine's outputs, the true-peak bound at every output rate measured independently of the
oracle, loudness targets reached, the neutral case, bitwise batch / order / EV_PDL=0 independence, mixed MicroBatcher requests,
and argument errors.

True-peak margins.  Each output's true peak is read at its own rate, oversampled to >= 192 kHz by resample_poly in fp64.  At
16 kHz and above the bound is C + 0.05 dB: resample_poly's default filter has at most 0.018 dB passband ripple up to 0.8 of
Nyquist, and a 12x reading of a full-scale tone up to 7.6 kHz reads at most 0.006 dB low.  One exception is measured, not
hidden: an item that starts or ends at full scale (the 45-degree sine, the +-1 sequence) is cut off by the resampler's output
itself, and that new edge rings in the first and last EDGE_S of a resampled output: 0.17 dB was measured at 24 kHz (on an
H100 80GB HBM3 at 700 W; the limiter's arithmetic does not depend on the card), so the whole output is held to RESAMPLED_EDGE
and the interior keeps the 0.05 dB bound.  The engine's outputs under a large loudness gain start loud too.  Below 16 kHz the
detector sees the low-passed signal at 16 kHz, but the output at 8 or 11.025 kHz also carries the resampler's transition band
folded back below its Nyquist rate, which the detector does not model: 0.01 dB was measured at 8 kHz and 0.37 dB at 11.025 kHz
(a voiced item with harmonics near 5.5 kHz; full-band noise reaches 0.45 dB in the oracle), so the bound there is
C + LOW_RATE_MARGIN[rate].

Loudness reached.  Two passes bring the voiced items of peak-to-loudness ratio 12 and 16 dB within 0.5 LU of -23, -16 and
-14 LUFS under a -1 dBTP ceiling.  At a ratio near 19 dB they do not at -16 and -14 LUFS: that case is asserted only at -23 and
the figures are printed, as they are at -10 LUFS, with no bound.  torchaudio's meter reads these
signals 0.12-0.22 LU below the BS.1770 oracle, hence TORCHAUDIO_LU."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audio_cases import SR, abi_limit, abi_loudness, engine_outputs, out_dict, padded_batch, ten_minutes
from conftest import ROOT
from emotivoice_b200 import _abi, audio, synth
from emotivoice_b200 import frontdoor as fd
from oracle import flac_oracle, limiter_oracle as O, loudness_oracle
from test_limiter import sine_45, voiced

pytestmark = pytest.mark.gpu
RATES = {16000: (1, 1), 22050: (441, 320), 24000: (3, 2), 44100: (441, 160), 48000: (3, 1), 8000: (1, 2), 11025: (441, 640)}
MARGIN = 0.05
RESAMPLED_EDGE, EDGE_S = 0.2, 0.002
TORCHAUDIO_LU = 0.3
LOW_RATE_MARGIN = {8000: 0.1, 11025: 0.5}
ENV_DB, REL = 1e-4, 1e-5


def synthetic_items():
    imp = np.zeros(SR, np.float32)
    imp[SR // 3] = 1.0
    sig = {"sine_45": sine_45(), "pm_one": np.tile(np.array([1, 1, -1, -1], np.float32), SR // 4), "impulse": imp,
           "voiced12": voiced(12.0), "voiced16": voiced(16.0, seed=1), "voiced20": voiced(20.0, seed=2),
           "silence": np.zeros(2 * SR, np.float32), "short": voiced(16.0, seed=3)[:5000]}
    return sig


def _compare(y, x, g, yo, Go, name):
    """GPU samples y against the oracle's yo / Go, and the envelope implied by y."""
    assert len(y) == len(x) == len(yo)
    err = np.abs(y.astype(np.float64) - yo) / np.maximum(np.abs(yo.astype(np.float64)), 1e-30)
    assert np.all(err <= REL), (name, err.max())
    xg = x.astype(np.float64) * g
    sel = np.abs(xg) > 1e-3
    if sel.any():
        G = 20 * np.log10(y[sel].astype(np.float64) / xg[sel])
        assert np.max(np.abs(G - Go[sel])) <= ENV_DB, (name, np.max(np.abs(G - Go[sel])))


def _two_pass_abi(lib, dev, w, lens, rate, ceiling, target):
    """The format_audio chain through the ABI: L0, pass 1, L1 of its result, pass 2 -> (out, L0, L1) host arrays."""
    L0 = abi_loudness(lib, dev, w, lens, target=target)[0]
    y1 = abi_limit(lib, dev, w, lens, rate, ceiling, L0, None, target)
    L1 = abi_loudness(lib, dev, y1[:, None, :].copy(), lens, target=target)[0]
    y2 = abi_limit(lib, dev, w, lens, rate, ceiling, L0, L1, target)
    return y1, y2, L0, L1


@pytest.mark.parametrize("rate", [16000, 8000])
def test_synthetic_items_match_the_oracle(model, lib, dev, rate):
    sig = synthetic_items()
    w, lens = padded_batch(list(sig.values()))
    for C, target in ((-1.0, None), (-1.0, -16.0), (-3.0, -23.0)):
        if target is None:
            y = abi_limit(lib, dev, w, lens, rate, C)
            for b, (name, x) in enumerate(sig.items()):
                yo, Go, _ = O.limit(x, SR, rate, C, 1.0)
                _compare(y[b, :lens[b]], x, 1.0, yo, Go, (name, rate, C))
            continue
        y1, y2, L0, L1 = _two_pass_abi(lib, dev, w, lens, rate, C, target)
        for b, (name, x) in enumerate(sig.items()):
            g1, g2 = O.pregain(target, L0[b]), O.pregain(target, L0[b], L1[b])
            yo, Go, _ = O.limit(x, SR, rate, C, g1)
            _compare(y1[b, :lens[b]], x, g1, yo, Go, (name, rate, C, target, 1))
            yo, Go, _ = O.limit(x, SR, rate, C, g2)
            _compare(y2[b, :lens[b]], x, g2, yo, Go, (name, rate, C, target, 2))
            if rate == SR:                                 # format_audio at the model's rate is the ABI chain, bit for bit
                want = fd.fetch_audio(model, out_dict(w, lens, dev), None, "float32", items=[b], hop=1, loudness=target, true_peak=C)[0]
                assert np.array_equal(want.view(np.int32), y2[b, :lens[b]].view(np.int32)), name


def test_ten_minutes_matches_the_oracle(lib, dev):
    x = ten_minutes() * np.float32(8.0)            # loud enough that limiting runs all along the item
    w, lens = padded_batch([x])
    y = abi_limit(lib, dev, w, lens, SR, -1.0)
    yo, Go, _ = O.limit(x, SR, SR, -1.0, 1.0, fast=True)
    _compare(y[0, :lens[0]], x, 1.0, yo, Go, "ten_minutes")
    assert Go.min() < -1.0


def test_engine_outputs_match_the_oracle(model, lib, dev):
    for name in ("b1_t100", "b3_padded"):
        out, xs = engine_outputs(model, dev)[name]
        w = out["wav_predictions"].cpu().numpy()
        lens = [len(x) for x in xs]
        y1, y2, L0, L1 = _two_pass_abi(lib, dev, w, lens, SR, -1.0, -14.0)
        got = fd.fetch_audio(model, out, None, "float32", loudness=-14.0, true_peak=-1.0)
        pcm = fd.fetch_audio(model, out, None, "pcm16", loudness=-14.0, true_peak=-1.0)
        for b, x in enumerate(xs):
            g2 = O.pregain(-14.0, L0[b], L1[b])
            yo, Go, _ = O.limit(x, SR, SR, -1.0, g2)
            _compare(y2[b, :lens[b]], x, g2, yo, Go, (name, b))
            assert np.array_equal(got[b].view(np.int32), y2[b, :lens[b]].view(np.int32)), (name, b)
            po = np.trunc(np.clip(yo.astype(np.float64) * 32768.0, -32768, 32767)).astype(np.int64)
            assert np.abs(pcm[b].astype(np.int64) - po).max() <= 1, (name, b)
            print(name, b, "L0 %.3f L1 %.3f out %.3f LUFS, tp %.4f dBTP" % (L0[b], L1[b],
                  loudness_oracle.integrated_loudness(got[b].astype(np.float64), SR), O.true_peak_db(got[b], SR)))


def _excess(y, rate, C):
    """(true peak over the whole output, over its interior without EDGE_S at each end) minus C, dB."""
    return O.true_peak_db(y, rate) - C, O.true_peak_db(y, rate, EDGE_S) - C


def test_true_peak_bound_at_every_rate(model, dev):
    sig = synthetic_items()
    out_e, xs = engine_outputs(model, dev)["b3_padded"]
    w, lens = padded_batch(list(sig.values()))
    out = out_dict(w, lens, dev)
    worst, bad = {}, []
    for C in (-1.0, -3.0):
        for rate in RATES:
            for target in (None, -14.0):
                for enc in ("float32", "pcm16", "flac"):
                    if enc == "flac" and target is None:
                        continue
                    kw = dict(loudness=target, true_peak=C)
                    ys = fd.fetch_audio(model, out, rate, enc, hop=1, **kw)
                    ys_e = fd.fetch_audio(model, out_e, rate, enc, **kw)
                    for name, y in list(zip(sig, ys)) + [("b3_%d" % b, y) for b, y in enumerate(ys_e)]:
                        if enc == "flac":
                            y = flac_oracle.decode(y)[1]
                        if enc != "float32":
                            y = y.astype(np.float64) / 32768.0
                        if not len(y) or not np.any(y):
                            continue
                        whole, inner = _excess(y, rate, C)
                        w0, w1 = worst.get((rate, enc), (-np.inf, -np.inf))
                        worst[(rate, enc)] = (max(w0, whole), max(w1, inner))
                        if rate in LOW_RATE_MARGIN:
                            ok = whole <= LOW_RATE_MARGIN[rate]
                        elif rate == SR:
                            ok = whole <= MARGIN
                        else:
                            ok = inner <= MARGIN and whole <= RESAMPLED_EDGE
                        if not ok:
                            bad.append((name, C, rate, target, enc, round(whole, 4), round(inner, 4)))
    for key in sorted(worst):
        print("true peak over the ceiling at %s: whole %.4f dB, interior %.4f dB" % (key, *worst[key]))
    assert not bad, bad


@pytest.mark.parametrize("plr", [12.0, 16.0, 20.0])
def test_loudness_targets_are_reached(model, dev, plr):
    import torchaudio.functional as F
    x = voiced(plr, seconds=6.0, seed=int(plr))
    w, lens = padded_batch([x])
    out = out_dict(w, lens, dev)
    for target in (-23.0, -16.0, -14.0, -10.0):
        y = fd.fetch_audio(model, out, None, "float32", hop=1, loudness=target, true_peak=-1.0)[0]
        Ly = loudness_oracle.integrated_loudness(y.astype(np.float64), SR)
        ta = float(F.loudness(torch.from_numpy(y)[None], SR))
        capped = fd.fetch_audio(model, out, None, "float32", hop=1, loudness=target)[0]
        Lc = loudness_oracle.integrated_loudness(capped.astype(np.float64), SR)
        print("PLR %.0f target %.0f: limited %.3f LUFS (torchaudio %.3f), tp %.3f dBTP; sample-peak cap %.3f LUFS"
              % (plr, target, Ly, ta, O.true_peak_db(y, SR), Lc))
        assert abs(ta - Ly) <= TORCHAUDIO_LU
        assert Ly >= Lc - 1e-3                            # never quieter than the sample-peak capped gain
        if target == -10.0 or (plr == 20.0 and target > -23.0):
            continue                                      # reported, no bound (see the module docstring)
        assert abs(Ly - target) <= 0.5, (plr, target, Ly)


def test_neutral_case_is_the_uncapped_gain(model, lib, dev):
    x = voiced(16.0, seed=5) * np.float32(0.05)
    w, lens = padded_batch([x])
    L0 = abi_loudness(lib, dev, w, lens)[0][0]
    g = O.pregain(-30.0, L0)
    assert 20 * np.log10(g * O.detect(x, SR, SR).max()) < -1.5          # nothing to limit
    y = fd.fetch_audio(model, out_dict(w, lens, dev), None, "float32", hop=1, loudness=-30.0, true_peak=-1.0)[0]
    y2 = abi_limit(lib, dev, w, lens, SR, -1.0, [L0], [L0], -30.0)[0]
    sel = np.abs(x) > 1e-4
    ratio = y[sel].astype(np.float64) / x[sel]
    assert np.max(np.abs(ratio / ratio[0] - 1.0)) <= 1e-6
    assert abs(ratio[0] / g - 1.0) <= 1e-3


def test_batch_and_order_independence(model, lib, dev):
    sig = list(synthetic_items().values())
    w, lens = padded_batch(sig)
    order = list(range(len(sig)))[::-1]
    full = _two_pass_abi(lib, dev, w, lens, SR, -1.0, -16.0)[1]
    rev = abi_limit(lib, dev, w, lens, SR, -2.0, items=order)
    fwd = abi_limit(lib, dev, w, lens, SR, -2.0)
    out = out_dict(w, lens, dev)
    enc_all = {fmt: fd.fetch_audio(model, out, *fmt, hop=1, loudness=-16.0, true_peak=-1.0) for fmt in ((8000, "mulaw"), (None, "float32"),
                                                                                                       (24000, "flac"))}
    for b, x in enumerate(sig):
        wb, lb = padded_batch([x])
        alone = _two_pass_abi(lib, dev, wb, lb, SR, -1.0, -16.0)[1]
        assert np.array_equal(alone[0, :lb[0]].view(np.int32), full[b, :lens[b]].view(np.int32)), b
        assert np.array_equal(rev[order.index(b), :lens[b]].view(np.int32), fwd[b, :lens[b]].view(np.int32)), b
        for fmt, allv in enc_all.items():
            one = fd.fetch_audio(model, out_dict(wb, lb, dev), *fmt, hop=1, loudness=-16.0, true_peak=-1.0)[0]
            assert np.array_equal(one.view(np.uint8), allv[b].view(np.uint8)), (fmt, b)


def pdl_dump(path):
    """Limited outputs of a seeded batch through the ABI (run under EV_PDL=0 by the test below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    lib = _abi.load()
    dev = torch.device("cuda:0")
    sig = synthetic_items()
    w, lens = padded_batch([sig[k] for k in ("sine_45", "voiced16", "short", "silence")])
    y1, y2, _, _ = _two_pass_abi(lib, dev, w, lens, 8000, -1.0, -16.0)
    np.savez(path, y1=np.nan_to_num(y1), y2=np.nan_to_num(y2))


def test_bitwise_equal_with_pdl_off(tmp_path):
    here = str(tmp_path / "pdl_on.npz")
    pdl_dump(here)
    off = str(tmp_path / "pdl_off.npz")
    path = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, EV_PDL="0", PYTHONPATH=os.pathsep.join(path))
    subprocess.run([sys.executable, "-c", "import test_limiter_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=600)
    x, y = np.load(here), np.load(off)
    for k in ("y1", "y2"):
        assert np.array_equal(x[k].view(np.int32), y[k].view(np.int32)), k


def test_microbatcher_mixed_ceilings_equal_fetch_audio_alone(model, dev):
    rng = np.random.default_rng(43)
    utts = [synth.make_utterance(rng, int(n)) for n in (14, 33, 9, 21, 17, 26, 12)]
    fmts = [(None, None, -16.0, -1.0), (8000, "mulaw", -16.0, -1.0), (24000, "float32", None, -3.0), (None, "flac", -14.0, -1.0),
            (None, None, -16.0, None), (24000, "pcm16", -16.0, -2.0), (None, None, None, None)]
    with fd.MicroBatcher(model, device=dev, max_batch=7, max_wait_s=0.5) as mb:
        futs = [mb.submit(u["ids"], int(u["speaker"]), u["style"], u["content"], sample_rate=r, encoding=e, loudness=t, true_peak=c)
                for u, (r, e, t, c) in zip(utts, fmts)]
        got = [f.result(timeout=120) for f in futs]
        assert mb.batches_run <= 2
    for u, (r, e, t, c), w in zip(utts, fmts, got):
        single = model(**fd.collate([(u["ids"], int(u["speaker"]), u["style"], u["content"])], dev))
        if r is None and e is None and t is None and c is None:
            assert torch.equal(single["wav_predictions"][0, 0].cpu(), w)
        else:
            want = fd.fetch_audio(model, single, r, "pcm16" if e is None else e, loudness=t, true_peak=c)[0]
            assert w.dtype == want.dtype and np.array_equal(w, want), (r, e, t, c)


def test_invalid_arguments_raise_before_anything_is_enqueued(model, lib, dev):
    out, xs = engine_outputs(model, dev)["b3_padded"]
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    for bad in (float("nan"), float("inf"), 1.0, -21.0, True, "-1"):
        with pytest.raises(ValueError):
            model.format_audio(out, 24000, "pcm16", loudness=-16.0, true_peak=bad)
        with pytest.raises(ValueError):
            fd.fetch_audio(model, out, true_peak=bad)
    w = out["wav_predictions"]
    n_in = torch.tensor([len(x) for x in xs], dtype=torch.int64, device=dev)
    bank, hold = audio.limit_bank(SR, SR)
    bank = torch.from_numpy(bank).to(dev)
    L = audio.limit_lookahead(SR)
    dst = torch.empty((3, w.stride(0)), dtype=torch.float32, device=dev)
    nb = lib.ev_limit_workspace_bytes(3, w.stride(0), L)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    lufs = torch.full((3,), -20.0, dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    rho = audio.limit_release(SR)

    def call(wp=w.data_ptr(), n=3, sr=SR, l0=None, l1=None, target=-23.0, C=-1.0, bp=bank.data_ptr(), ph=bank.shape[0], taps=bank.shape[1],
             la=L, hd=hold, rel=rho, op=dst.data_ptr(), ostride=dst.stride(0), wsb=nb):
        return lib.ev_limit(wp, w.stride(0), n_in.data_ptr(), None, n, sr, l0, l1, target, C, bp, ph, taps, la, hd, rel, op, ostride,
                            ws.data_ptr(), wsb, st)

    for kw in (dict(wp=None), dict(bp=None), dict(op=None), dict(n=0), dict(n=65536), dict(sr=3999), dict(C=0.5), dict(C=-20.5),
               dict(C=float("nan")), dict(l0=lufs.data_ptr(), target=1.0), dict(l1=lufs.data_ptr()), dict(taps=20), dict(ph=0),
               dict(hd=hold - 1 if hold else -1), dict(la=2000), dict(rel=0.0), dict(rel=rho * 1.0000001), dict(ostride=w.stride(0) - 1),
               dict(wsb=nb - 1)):
        assert call(**kw) == -1, kw
    assert lib.ev_limit_workspace_bytes(0, w.stride(0), L) == 0 and lib.ev_limit_workspace_bytes(3, w.stride(0), 5000) == 0
    assert _abi.launch_count() == n0
    assert call(l0=lufs.data_ptr(), l1=lufs.data_ptr()) == 0
    assert _abi.launch_count() == n0 + 3
