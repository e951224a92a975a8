"""Loudness normalisation on the GPU (``JETSGenerator.measure_loudness``, ``format_audio(loudness=...)``, ev_loudness and
the gain of ev_format_audio): integrated loudness and peak against the fp64 BS.1770-4 oracle on the engine's outputs and on
synthetic items with NaN past their lengths, batch independence, the gain identity of every encoding, the normalised result, no
change without a target or under unit gains (and with EV_PDL=0), mixed targets in one MicroBatcher forward, and argument
errors."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audio_cases import SR, abi_loudness, engine_outputs, out_dict, padded_batch, ten_minutes
from conftest import GOLDEN, ROOT
from emotivoice_b200 import _abi, audio, synth
from emotivoice_b200 import frontdoor as fd
from oracle import loudness_oracle as O

pytestmark = pytest.mark.gpu
DL = 1e-3                   # LU
CEILING = 10.0 ** (-1.0 / 20.0)


def _sine(dbfs, seconds, f):
    n = np.arange(int(round(seconds * SR)))
    return 10.0 ** (dbfs / 20.0) * np.sin(2 * np.pi * f * n / SR)


def _noise(dbfs, n, seed):
    return np.clip(10.0 ** (dbfs / 20.0) * np.random.default_rng(seed).standard_normal(n), -1.0, 1.0)


def synthetic_items():
    """name -> float32 signal: tones, EBU Tech 3341 case 5 in mono, noise at three levels, the block-count edges, a length that
    ends inside a sub-block, silence."""
    sig = {
        "tone_997_m20": _sine(-20, 5, 997.0),
        "tone_100_m6": _sine(-6, 3, 100.0),
        "case5": np.concatenate([_sine(-36, 10, 1000.0), _sine(-23, 60, 1000.0), _sine(-36, 10, 1000.0)]),
        "noise_m10": _noise(-10, 3 * SR, 1),
        "noise_m40": _noise(-40, 3 * SR, 2),
        "noise_m65": _noise(-65, 3 * SR, 3),
        "n6399": _noise(-20, 6399, 4),
        "n6400": _noise(-20, 6400, 5),
        "n6401": _noise(-20, 6401, 6),
        "n32777": _noise(-25, 2 * SR + 777, 7) + _sine(-30, (2 * SR + 777) / SR, 440.0),
        "silence": np.zeros(2 * SR),
    }
    return {k: v.astype(np.float32) for k, v in sig.items()}


def gate_margin(x):
    """Smallest distance (LU) of a block's loudness to the absolute or relative gate (inf without blocks)."""
    _, l, rel = O.gating(np.asarray(x, np.float64), SR)
    l = l[np.isfinite(l)]
    if not len(l):
        return np.inf
    m = np.abs(l + 70.0).min()
    return m if not np.isfinite(rel) else min(m, np.abs(l - rel).min())


def _oracle(x, target):
    L = O.integrated_loudness(np.asarray(x, np.float64), SR)
    pk = O.peak(x)
    return L, pk, O.gain(L, pk, target)


def _check(L, pk, x, name):
    Lo, po, _ = _oracle(x, -23.0)
    assert pk == np.float32(po), (name, pk, po)
    if np.isfinite(Lo):
        assert gate_margin(x) > 0.01, name
        assert abs(float(L) - Lo) <= DL, (name, L, Lo)
    else:
        assert L == -np.inf, (name, L)


def test_engine_outputs_match_the_oracle(model, dev, lib):
    for name, (out, xs) in engine_outputs(model, dev).items():
        lufs, pk = model.measure_loudness(out)
        assert lufs.dtype == torch.float32 and lufs.device == dev and lufs.shape == (len(xs),)
        lufs, pk = lufs.cpu().numpy(), pk.cpu().numpy()
        for b, x in enumerate(xs):
            _check(lufs[b], pk[b], x, (name, b))
        print(name, "lufs", lufs.tolist(), "peak", pk.tolist())
    lufs, pk = model.measure_loudness(engine_outputs(model, dev)["b3_padded"][0], items=[2, 0])
    whole = model.measure_loudness(engine_outputs(model, dev)["b3_padded"][0])
    assert torch.equal(lufs, whole[0][[2, 0]]) and torch.equal(pk, whole[1][[2, 0]])


def test_synthetic_items_match_the_oracle(lib, dev):
    sig = synthetic_items()
    w, lens = padded_batch(list(sig.values()))
    lufs, pk, _ = abi_loudness(lib, dev, w, lens)
    for b, (name, x) in enumerate(sig.items()):
        _check(lufs[b], pk[b], x, name)
    assert lufs[list(sig).index("n6399")] == -np.inf and lufs[list(sig).index("silence")] == -np.inf
    assert np.isfinite(lufs[list(sig).index("n6400")])
    x = ten_minutes()
    w, lens = padded_batch([x])
    lufs, pk, _ = abi_loudness(lib, dev, w, lens)
    _check(lufs[0], pk[0], x, "ten_minutes")


def test_batch_independence(model, lib, dev):
    sig = list(synthetic_items().values())
    w, lens = padded_batch(sig)
    full = abi_loudness(lib, dev, w, lens, target=-20.0)
    order = list(range(len(sig)))[::-1]
    rev = abi_loudness(lib, dev, w, lens, items=order, target=-20.0)
    out = out_dict(w, lens, dev)
    enc_all = {fmt: fd.fetch_audio(model, out, *fmt, hop=1, loudness=-20.0) for fmt in ((8000, "mulaw"), (None, "float32"))}
    for b, x in enumerate(sig):
        wb, lb = padded_batch([x])
        alone = abi_loudness(lib, dev, wb, lb, target=-20.0)
        for a, f, r in zip(alone, full, rev):
            assert a.view(np.int32)[0] == f.view(np.int32)[b] == r.view(np.int32)[order.index(b)], b
        for fmt, allv in enc_all.items():
            one = fd.fetch_audio(model, out_dict(wb, lb, dev), *fmt, hop=1, loudness=-20.0)[0]
            assert np.array_equal(one.view(np.uint8), allv[b].view(np.uint8)), (fmt, b)


def _g711():
    z = np.load(GOLDEN + "/g711.npz")
    return {"mulaw": z["ulaw"], "alaw": z["alaw"]}


@pytest.mark.parametrize("target", [-30.0, -16.0])
def test_gain_identity_and_result(model, lib, dev, target):
    out, xs = engine_outputs(model, dev)["b1_t100"]
    x = xs[0]
    w = out["wav_predictions"].cpu().numpy()
    _, _, g = abi_loudness(lib, dev, w, [len(x)], target=target)
    g = g[0]
    Lo, po, go = _oracle(x, target)
    assert abs(g / go - 1) <= 10.0 ** (DL / 20.0) - 1.0
    tables = _g711()
    for rate in (16000, 24000, 8000):
        plain = fd.fetch_audio(model, out, rate, "float32")[0]
        y = fd.fetch_audio(model, out, rate, "float32", loudness=target)[0]
        want = (plain * np.float32(g)).astype(np.float32)
        assert np.array_equal(y.view(np.int32), want.view(np.int32)), rate
        pcm = np.trunc(np.clip(want.astype(np.float64) * 32768.0, -32768, 32767)).astype(np.int16)
        assert np.array_equal(fd.fetch_audio(model, out, rate, "pcm16", loudness=target)[0], pcm)
        for enc in ("mulaw", "alaw"):
            assert np.array_equal(fd.fetch_audio(model, out, rate, enc, loudness=target)[0], tables[enc][pcm.astype(np.int64) + 32768])
        if rate == 16000:
            Ly = O.integrated_loudness(y.astype(np.float64), SR)
            if 10.0 ** ((target - Lo) / 20.0) * po < CEILING:      # -30 LUFS: g ~ 7.4, the peak stays below the ceiling
                assert target == -30.0 and abs(Ly - target) <= 0.01, Ly
            else:                                    # -16 LUFS: the -1 dBFS ceiling binds
                assert target == -16.0 and Ly < target and abs(np.abs(y).max() - CEILING) <= 1e-6, (Ly, np.abs(y).max())
    print("b1_t100 target %.1f: oracle L %.3f peak %.4f g %.6f" % (target, Lo, po, g))


def test_silence_and_short_items_are_left_as_they_are(model, dev):
    sig = synthetic_items()
    w, lens = padded_batch([sig["silence"], sig["n6399"], sig["n6400"]])
    out = out_dict(w, lens, dev)
    for fmt in ((None, "float32"), (24000, "pcm16")):
        plain = fd.fetch_audio(model, out, *fmt, hop=1)
        norm = fd.fetch_audio(model, out, *fmt, hop=1, loudness=-23.0)
        assert np.array_equal(plain[0].view(np.uint8), norm[0].view(np.uint8))
        assert np.array_equal(plain[1].view(np.uint8), norm[1].view(np.uint8))
        assert not np.array_equal(plain[2], norm[2])


def pdl_dump(path):
    """L, g and the gain-formatted outputs of a seeded batch, straight through the ABI (run under EV_PDL=0 by the test below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    lib = _abi.load()
    dev = torch.device("cuda:0")
    sig = synthetic_items()
    w, lens = padded_batch([sig[k] for k in ("tone_997_m20", "noise_m40", "n32777", "silence")])
    lufs, pk, g = abi_loudness(lib, dev, w, lens, target=-18.0)
    wt = torch.from_numpy(w).to(dev)
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    offs = audio.packed_offsets(lens, range(len(lens)), 3, 2)
    off = torch.from_numpy(offs[:-1]).to(dev)
    bank = torch.from_numpy(audio.polyphase_bank(3, 2)).to(dev)
    gain = torch.from_numpy(g).to(dev)
    dst = torch.empty(int(offs[-1]), dtype=torch.float32, device=dev)
    _abi.check(lib.ev_format_audio(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None, len(lens), off.data_ptr(), bank.data_ptr(),
                                   3, 2, bank.shape[1], 0, dst.data_ptr(), gain.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    np.savez(path, lufs=lufs, peak=pk, gain=g, out=dst.cpu().numpy())


def test_no_change_without_a_target_and_with_pdl_off(model, lib, dev, tmp_path):
    out, xs = engine_outputs(model, dev)["b3_padded"]
    w = out["wav_predictions"]
    n_in = torch.tensor([len(x) for x in xs], dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    for up, down, enc in ((1, 1, 1), (3, 2, 0), (1, 2, 2), (441, 320, 3)):
        bank = None if (up, down) == (1, 1) else torch.from_numpy(audio.polyphase_bank(up, down)).to(dev)
        offs = audio.packed_offsets([len(x) for x in xs], [2, 0, 1], up, down)
        off = torch.from_numpy(offs[:-1]).to(dev)
        it = torch.tensor([2, 0, 1], dtype=torch.int64, device=dev)
        a = torch.full((int(offs[-1]) * 4,), 7, dtype=torch.uint8, device=dev)
        b = a.clone()
        ones = torch.ones(3, dtype=torch.float32, device=dev)
        args = (w.data_ptr(), w.stride(0), n_in.data_ptr(), it.data_ptr(), 3, off.data_ptr(), None if bank is None else bank.data_ptr(),
                up, down, 0 if bank is None else bank.shape[1], enc)
        _abi.check(lib.ev_format_audio(*args, a.data_ptr(), None, st))
        _abi.check(lib.ev_format_audio(*args, b.data_ptr(), ones.data_ptr(), st))       # fp32(y * 1) == y
        assert torch.equal(a, b), (up, down, enc)
    here = str(tmp_path / "pdl_on.npz")
    pdl_dump(here)
    off = str(tmp_path / "pdl_off.npz")
    path = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, EV_PDL="0", PYTHONPATH=os.pathsep.join(path))
    subprocess.run([sys.executable, "-c", "import test_loudness_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=600)
    x, y = np.load(here), np.load(off)
    for k in ("lufs", "peak", "gain", "out"):
        assert np.array_equal(x[k].view(np.int32), y[k].view(np.int32)), k


def test_microbatcher_mixed_targets_equal_fetch_audio_alone(model, dev):
    rng = np.random.default_rng(41)
    utts = [synth.make_utterance(rng, int(n)) for n in (14, 33, 9, 21, 17, 26)]
    fmts = [(None, None, -23.0), (8000, "mulaw", -16.0), (24000, "float32", -30.0), (None, "alaw", -23.0), (24000, "pcm16", None),
            (None, None, None)]
    with fd.MicroBatcher(model, device=dev, max_batch=6, max_wait_s=0.5) as mb:
        futs = [mb.submit(u["ids"], int(u["speaker"]), u["style"], u["content"], sample_rate=r, encoding=e, loudness=t)
                for u, (r, e, t) in zip(utts, fmts)]
        got = [f.result(timeout=120) for f in futs]
        assert mb.batches_run <= 2
    for u, (r, e, t), w in zip(utts, fmts, got):
        single = model(**fd.collate([(u["ids"], int(u["speaker"]), u["style"], u["content"])], dev))
        if r is None and e is None and t is None:
            assert torch.equal(single["wav_predictions"][0, 0].cpu(), w)
        else:
            want = fd.fetch_audio(model, single, r, "pcm16" if e is None else e, loudness=t)[0]
            assert w.dtype == want.dtype and np.array_equal(w, want), (r, e, t)


def test_invalid_arguments_raise_before_anything_is_enqueued(model, lib, dev):
    out, xs = engine_outputs(model, dev)["b3_padded"]
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    for bad in (float("nan"), float("inf"), 1.0, -71.0, True, "-23"):
        with pytest.raises(ValueError):
            model.format_audio(out, 24000, "pcm16", loudness=bad)
        with pytest.raises(ValueError):
            fd.fetch_audio(model, out, loudness=bad)
    with pytest.raises(ValueError):
        model.measure_loudness(out, items=[3])
    w = out["wav_predictions"]
    n_in = torch.tensor([len(x) for x in xs], dtype=torch.int64, device=dev)
    res = torch.empty((3, 3), dtype=torch.float32, device=dev)
    kc = audio.k_weighting(SR)
    nb = lib.ev_loudness_workspace_bytes(3, w.stride(0), SR)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def call(wp=w.data_ptr(), n=3, sr=SR, kcp=kc.ctypes.data, target=-23.0, lufs=res[0].data_ptr(), wsb=nb):
        return lib.ev_loudness(wp, w.stride(0), n_in.data_ptr(), None, n, sr, kcp, target, lufs, res[1].data_ptr(), res[2].data_ptr(),
                               ws.data_ptr(), wsb, st)

    for kw in (dict(wp=None), dict(kcp=None), dict(lufs=None), dict(n=0), dict(n=65536), dict(sr=16005), dict(sr=16001),
               dict(target=1.0), dict(target=float("nan")), dict(wsb=nb - 1)):
        assert call(**kw) == -1, kw
    assert lib.ev_loudness_workspace_bytes(3, w.stride(0), 16005) == 0
    assert _abi.launch_count() == n0
    assert call() == 0
    assert _abi.launch_count() == n0 + 2
