"""The loudness meter on the GPU (``loudness.meter``, ``JETSGenerator.meter``, ev_meter): every result against the fp64 oracle
(``oracle/meter_oracle.py``) at 8, 16, 22.05, 24, 44.1, 48 and 96 kHz on items around the window lengths, silence, speech-like
signals and the engine's outputs, and at 4 and 192 kHz; I bitwise ev_loudness's lufs; bitwise batch, order and EV_PDL=0 independence; the limiter
and format_audio unchanged beside it; the metered output chain; a one-hour 48 kHz recording; launch counts and argument
errors."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from numpy.lib.stride_tricks import sliding_window_view
from scipy.signal import lfilter, resample_poly

from audio_cases import abi_limit, engine_outputs, padded_batch
from conftest import ROOT
from emotivoice_b200 import _abi, audio, loudness
from oracle import limiter_oracle
from oracle import meter_oracle as O
from test_watermark import speech_like

pytestmark = pytest.mark.gpu
DL = 1e-3                   # LU: the tolerance of test_loudness_gpu, plus each value's own K-coefficient allowance (below)
DTP = 1e-4                  # dB
GATE = -70.0                # LUFS: values under the absolute gate enter no gated result and are compared only as being under
                            # it (a window holding only the K-filter's ringing after much louder content is filtered in fp32
                            # relative to that content, and reads up to ~0.02 LU off there)
RATES = (8000, 16000, 22050, 24000, 44100, 48000, 96000)
_worst = {"loudness_lu": 0.0, "loudness_lu_over_allowance": 0.0, "allowance_lu": 0.0, "true_peak_db": 0.0}


def _noise(sr, dbfs, n, seed):
    return np.clip(10.0 ** (dbfs / 20.0) * np.random.default_rng(seed).standard_normal(n), -1.0, 1.0)


def _tone(sr, dbfs, n, f):
    return 10.0 ** (dbfs / 20.0) * np.sin(2 * np.pi * f * np.arange(n) / sr)


def items_at(sr):
    """name -> float32 signal at sr: the window-length edges, a partial last sub-block, silence, speech-like signals."""
    S = sr // 10
    speech = resample_poly(speech_like(12.0, 5, 0.7), sr, 16000) if sr != 16000 else speech_like(12.0, 5, 0.7)
    sig = {
        "under_400ms": _noise(sr, -20, 4 * S - 1, 1),
        "400ms": _noise(sr, -20, 4 * S, 2),
        "under_3s": _noise(sr, -24, 30 * S - 1, 3) + _tone(sr, -30, 30 * S - 1, 440.0),
        "3s": _noise(sr, -24, 30 * S, 4),
        "partial": np.concatenate([_tone(sr, -30, 20 * S, 1000.0), _noise(sr, -18, 35 * S + 17, 5)]),
        "zeros": np.zeros(25 * S),
        "speech": speech,
        "speech_quiet_tail": np.concatenate([speech[:6 * sr] * 0.5, speech[6 * sr:] * 0.05]),
    }
    return {k: v.astype(np.float32) for k, v in sig.items()}


def _margin(st):
    """Smallest distance (LU) of a short-term value to either gate of the loudness range (inf without values)."""
    s = np.asarray(st, np.float64)
    s = s[np.isfinite(s)]
    if not len(s):
        return np.inf
    m = np.abs(s + 70.0).min()
    s = s[s > -70.0]
    if len(s):
        m = min(m, np.abs(s - (10.0 * np.log10(np.mean(10.0 ** (s / 10.0))) - 20.0)).min())
    return m


def fp32_coefficient_levels(x, sr):
    """I, M, S and LRA in fp64 with the K-weighting coefficients rounded to fp32, as the kernels filter.  Their distance to
    the oracle is what that rounding alone moves each value: 6e-5 LU at 16 kHz, 2e-5 at 48 kHz, 1.7e-3 at 96 kHz on speech,
    where the 38 Hz high-pass's poles sit closest to 1."""
    k = audio.k_weighting(sr).astype(np.float32).astype(np.float64)
    y = lfilter(k[5:8], [1.0, k[8], k[9]], lfilter(k[0:3], [1.0, k[3], k[4]], np.asarray(x, np.float64)))
    S = sr // 10
    nf = len(y) // S
    e = (y[:nf * S] ** 2).reshape(nf, S).sum(axis=1)

    def windows(blocks):
        if nf < blocks:
            return np.zeros(0), np.zeros(0)
        z = sliding_window_view(e, blocks).sum(axis=1) / (blocks * S)
        with np.errstate(divide="ignore"):
            return z, -0.691 + 10.0 * np.log10(z)

    z, m = windows(4)
    keep = m > -70.0
    I = -np.inf
    if keep.any():
        keep &= m > -0.691 + 10.0 * np.log10(z[keep].mean()) - 10.0
        if keep.any():
            I = -0.691 + 10.0 * np.log10(z[keep].mean())
    st = windows(30)[1]
    return dict(integrated=I, momentary=m, short_term=st, loudness_range=O.loudness_range(None, sr, st),
                max_momentary=float(np.max(m, initial=-np.inf)), max_short_term=float(np.max(st, initial=-np.inf)))


def _host(m, b=None):
    """Meter -> dict of host values (item b, or all)."""
    out = {}
    for k in m._fields:
        v = getattr(m, k)
        if v is not None:
            v = v.cpu().numpy()
            out[k] = v if b is None else v[b]
    return out


def _close(got, want, rounded, name):
    """got (GPU, float32) against the fp64 oracle: within DL plus what rounding the coefficients moves the value, where the
    oracle is above the absolute gate; under it where the oracle is."""
    got, want, rounded = (np.atleast_1d(np.asarray(v, np.float64)) for v in (got, want, rounded))
    loud = want > GATE
    assert np.all(got[~loud] <= GATE + DL), (name, got[~loud].max())
    if loud.any():
        err, allow = np.abs(got[loud] - want[loud]), np.abs(rounded[loud] - want[loud])
        assert np.all(err <= DL + allow), (name, (err - allow).max(), err.max())
        _worst["loudness_lu"] = max(_worst["loudness_lu"], float(err.max()))
        _worst["loudness_lu_over_allowance"] = max(_worst["loudness_lu_over_allowance"], float((err - allow).max()))
        _worst["allowance_lu"] = max(_worst["allowance_lu"], float(allow.max()))


def check_against_oracle(got, x, sr, name, true_peak=None):
    """got: host values of one item; x its samples.  ``true_peak``: the oracle's value, when computed apart."""
    o = O.meter(np.asarray(x, np.float64), sr, true_peak=true_peak is None)
    r = fp32_coefficient_levels(x, sr)
    tp = o["true_peak"] if true_peak is None else true_peak
    assert got["sample_peak"] == np.float32(o["sample_peak"]), (name, got["sample_peak"], o["sample_peak"])
    for k in ("integrated", "max_momentary", "max_short_term"):
        if np.isfinite(o[k]):
            _close(got[k], o[k], r[k], (name, k))
        else:
            assert got[k] == -np.inf, (name, k, got[k], o[k])
    if np.isfinite(tp):
        assert abs(float(got["true_peak"]) - tp) <= DTP, (name, got["true_peak"], tp)
        _worst["true_peak_db"] = max(_worst["true_peak_db"], abs(float(got["true_peak"]) - tp))
    else:
        assert got["true_peak"] == -np.inf, (name, got["true_peak"])
    if math.isnan(o["loudness_range"]):
        assert math.isnan(got["loudness_range"]), (name, got["loudness_range"])
    elif _margin(o["short_term"]) > 0.01:
        assert abs(float(got["loudness_range"]) - o["loudness_range"]) <= DL + abs(r["loudness_range"] - o["loudness_range"]), (
            name, got["loudness_range"], o["loudness_range"])
    for k in ("momentary", "short_term"):
        if k in got:
            assert np.all(np.isnan(got[k][len(o[k]):])), (name, k)
            _close(got[k][:len(o[k])], o[k], r[k], (name, k))
    return o


def _batch(sig, dev, poison=True):
    w, lens = padded_batch(list(sig), poison)
    return torch.from_numpy(w[:, 0]).to(dev), lens


def abi_lufs(lib, dev, wt, lens, sr):
    """ev_loudness's lufs of the rows of wt at sr (host float32)."""
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    k = len(lens)
    res = torch.empty((3, k), dtype=torch.float32, device=dev)
    kc = audio.k_weighting(sr)
    nb = lib.ev_loudness_workspace_bytes(k, wt.stride(0), sr)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_loudness(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None, k, sr, kc.ctypes.data, -23.0, res[0].data_ptr(),
                               res[1].data_ptr(), res[2].data_ptr(), ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    return res[0].cpu().numpy()


@pytest.mark.parametrize("sr", RATES)
def test_items_match_the_oracle_and_ev_loudness(lib, dev, sr):
    sig = items_at(sr)
    wt, lens = _batch(sig.values(), dev)
    m = loudness.meter(wt, sr, lens, series=True)
    got = _host(m)
    for b, (name, x) in enumerate(sig.items()):
        check_against_oracle({k: v[b] for k, v in got.items()}, x, sr, (sr, name))
    lufs = abi_lufs(lib, dev, wt, lens, sr)
    assert np.array_equal(got["integrated"].view(np.int32), lufs.view(np.int32)), sr
    names = list(sig)
    for short in ("under_400ms", "zeros"):
        b = names.index(short)
        assert got["max_momentary"][b] == got["max_short_term"][b] == got["integrated"][b] == -np.inf
        assert math.isnan(got["loudness_range"][b])
    assert got["max_short_term"][names.index("under_3s")] == -np.inf and np.isfinite(got["max_momentary"][names.index("under_3s")])
    assert np.isfinite(got["max_short_term"][names.index("3s")]) and got["short_term"].shape[1] == max(lens) // (sr // 10) - 29
    print("worst so far:", _worst)


@pytest.mark.parametrize("sr", (4000, 192000))
def test_the_rate_range_edges(dev, sr):
    """4 kHz: the widest detector bank (48 phases); 192 kHz: no bank, the true peak is the sample peak."""
    S = sr // 10
    sig = {"noise": _noise(sr, -22, 47 * S + 5, 21), "tone": _tone(sr, -12, 31 * S, 0.23 * sr)}
    sig = {k: v.astype(np.float32) for k, v in sig.items()}
    wt, lens = _batch(sig.values(), dev)
    got = _host(loudness.meter(wt, sr, lens, series=True))
    for b, (name, x) in enumerate(sig.items()):
        check_against_oracle({k: v[b] for k, v in got.items()}, x, sr, (sr, name))
    if sr == 192000:
        assert np.array_equal(got["true_peak"], (20 * np.log10(got["sample_peak"].astype(np.float64))).astype(np.float32))


def test_engine_outputs_match_the_oracle(model, dev):
    for name, (out, xs) in engine_outputs(model, dev).items():
        m = _host(model.meter(out, series=True))
        for b, x in enumerate(xs):
            check_against_oracle({k: v[b] for k, v in m.items()}, x, 16000, (name, b))
        one = model.meter(out, items=[len(xs) - 1])
        assert torch.equal(one.integrated, model.measure_loudness(out, items=[len(xs) - 1])[0])
    print("worst:", _worst)


def test_results_do_not_depend_on_the_batch_or_its_order(dev):
    sr = 22050
    sig = list(items_at(sr).values())
    wt, lens = _batch(sig, dev)
    full = _host(loudness.meter(wt, sr, lens, series=True))
    rev = _host(loudness.meter(wt.flip(0), sr, lens[::-1], series=True))
    B = len(sig)
    for b, x in enumerate(sig):
        wb, lb = _batch([x], dev, poison=False)
        alone = _host(loudness.meter(wb, sr, lb, series=True), 0)
        for k, v in alone.items():
            a, f, r = np.asarray(v), full[k][b], rev[k][B - 1 - b]
            if k in ("momentary", "short_term"):
                n = len(a)
                assert np.array_equal(a.view(np.int32), f[:n].view(np.int32)) and np.array_equal(a.view(np.int32), r[:n].view(np.int32)), (b, k)
            else:
                assert a.view(np.int32) == f.view(np.int32) == r.view(np.int32), (b, k, a, f, r)


def test_packed_outputs_are_read_in_place(model, dev):
    out, xs = engine_outputs(model, dev)["b3_padded"]
    for rate in (16000, 24000, 48000, 8000):
        packed, offs = model.format_audio(out, rate, "float32", items=[2, 0, 1])
        host = packed.cpu().numpy()
        m = _host(model.meter(out, rate, items=[2, 0, 1], series=True))
        wt, lens = _batch([host[offs[k]:offs[k + 1]] for k in range(3)], dev)
        want = _host(loudness.meter(wt, rate, lens, series=True))
        for k in m:
            if k in ("momentary", "short_term"):
                c = min(m[k].shape[1], want[k].shape[1])
                assert np.array_equal(m[k][:, :c].view(np.int32), want[k][:, :c].view(np.int32)), (rate, k)
            else:
                assert np.array_equal(m[k].view(np.int32), want[k].view(np.int32)), (rate, k)


def test_metered_chain_agrees_with_the_oracle_on_what_format_audio_delivers(model, dev):
    """model.meter(loudness=-23, true_peak=-1) against the oracle on the host copy of format_audio's float32 output; what it
    reads is printed, not held to the targets (the limiter bounds the true peak at the model's rate, before resampling)."""
    for name in ("b1_t100", "b3_padded"):
        out, _ = engine_outputs(model, dev)[name]
        for rate in (16000, 24000, 48000):
            m = _host(model.meter(out, sample_rate=rate, loudness=-23, true_peak=-1))
            packed, offs = model.format_audio(out, rate, "float32", loudness=-23, true_peak=-1)
            y = packed.cpu().numpy()
            for k in range(len(offs) - 1):
                check_against_oracle({f: v[k] for f, v in m.items()}, y[offs[k]:offs[k + 1]], rate, (name, rate, k))
                print("%s[%d] at %d Hz, loudness -23 true_peak -1: I %.3f LUFS, true peak %.3f dBTP, LRA %.2f LU, max M %.2f, max S %.2f"
                      % (name, k, rate, m["integrated"][k], m["true_peak"][k], m["loudness_range"][k], m["max_momentary"][k],
                         m["max_short_term"][k]))


def _limit_and_format(model, dev):
    """ev_limit of a seeded batch and format_audio of the fixture outputs (with loudness, true peak and a watermark)."""
    sig = [speech_like(3.0, 11), speech_like(2.3, 12, 0.9)]
    w, lens = padded_batch(sig)
    lim = abi_limit(_abi.load(), dev, w, lens, 24000, -1.0)
    out, _ = engine_outputs(model, dev)["b3_padded"]
    fmt = model.format_audio(out, 48000, "pcm16", loudness=-16, true_peak=-1, watermark=7)[0].cpu().numpy()
    return np.nan_to_num(lim, nan=7.0), fmt


def chain_dump(path, with_meter):
    from emotivoice_b200 import build, synth
    from emotivoice_b200.config import default_config
    from emotivoice_b200.modules import JETSGenerator
    build.build(verbose=False)
    dev = torch.device("cuda:0")
    conf = default_config()
    model = JETSGenerator(conf).to(dev)
    model.load_state_dict(synth.make_state_dict(conf))
    model.eval()
    if with_meter:
        out, _ = engine_outputs(model, dev)["b3_padded"]
        model.meter(out, 48000, loudness=-16, true_peak=-1, watermark=7)
        loudness.meter(out["wav_predictions"][:, 0], 16000)
    lim, fmt = _limit_and_format(model, dev)
    np.savez(path, lim=lim, fmt=fmt)


def pdl_dump(path):
    """Meter results of a seeded batch (run under EV_PDL=0 by the test below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    dev = torch.device("cuda:0")
    sr = 44100
    wt, lens = _batch(items_at(sr).values(), dev)
    m = _host(loudness.meter(wt, sr, lens, series=True))
    np.savez(path, **m)


def _subprocess(expr, path, env_extra):
    py = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(py), **env_extra)
    subprocess.run([sys.executable, "-c", expr, path], env=env, check=True, cwd=ROOT, timeout=900)


def test_same_bits_with_pdl_off(tmp_path):
    here, off = str(tmp_path / "on.npz"), str(tmp_path / "off.npz")
    pdl_dump(here)
    _subprocess("import test_meter_gpu as T, sys; T.pdl_dump(sys.argv[1])", off, {"EV_PDL": "0"})
    x, y = np.load(here), np.load(off)
    assert sorted(x.files) == sorted(y.files)
    for k in x.files:
        assert np.array_equal(x[k].view(np.int32), y[k].view(np.int32)), k


def test_limiter_and_format_audio_are_unchanged_beside_the_meter(model, dev, tmp_path):
    never = str(tmp_path / "never.npz")
    _subprocess("import test_meter_gpu as T, sys; T.chain_dump(sys.argv[1], False)", never, {})
    here = str(tmp_path / "here.npz")
    chain_dump(here, True)
    x, y = np.load(never), np.load(here)
    assert np.array_equal(x["lim"].view(np.int32), y["lim"].view(np.int32))
    assert np.array_equal(x["fmt"], y["fmt"])


def one_hour(sr=48000):
    """60 minutes of noise whose level moves over 20 dB, with a minute of silence and a minute of quiet tone."""
    n = 3600 * sr
    rng = np.random.default_rng(60)
    x = rng.standard_normal(n).astype(np.float32)
    t = np.arange(n, dtype=np.float32) / np.float32(sr)
    x *= (10.0 ** ((-28.0 + 10.0 * np.sin(2 * np.pi * t / 613.0)) / 20.0)).astype(np.float32)
    x[600 * sr:660 * sr] = 0.0
    x[1200 * sr:1260 * sr] = (0.01 * np.sin(2 * np.pi * 1000.0 * t[:60 * sr])).astype(np.float32)
    return np.clip(x, -1.0, 1.0)


def true_peak_chunked(x, sr, chunk=1 << 22):
    """limiter_oracle.true_peak_db of a long signal, a chunk at a time: each chunk with 48 samples of context on either side,
    whose outputs are left out again."""
    m = 48
    xp = np.concatenate([np.zeros(m), np.asarray(x, np.float64), np.zeros(m)])
    best = -np.inf
    for a in range(0, len(x), chunk):
        b = min(len(x), a + chunk)
        best = max(best, limiter_oracle.true_peak_db(xp[a:b + 2 * m], sr, edge_s=m / sr))
    return best


def test_one_hour_at_48k(dev):
    sr = 48000
    x = one_hour(sr)
    wt = torch.from_numpy(x[None]).to(dev)
    torch.cuda.synchronize()
    m = _host(loudness.meter(wt, sr, series=True), 0)
    assert m["short_term"].shape == (36000 - 29,)
    tp = true_peak_chunked(x, sr)
    o = check_against_oracle(m, x, sr, "one_hour", true_peak=tp)
    print("one hour at 48 kHz: I %.3f (oracle %.3f) LRA %.3f (%.3f) max M %.3f max S %.3f true peak %.5f (%.5f)"
          % (m["integrated"], o["integrated"], m["loudness_range"], o["loudness_range"], m["max_momentary"], m["max_short_term"],
             m["true_peak"], tp))
    assert np.isfinite(m["loudness_range"]) and m["loudness_range"] > 10.0
    print("worst:", _worst)


def test_launch_counts_and_argument_errors(model, lib, dev):
    out, xs = engine_outputs(model, dev)["b3_padded"]
    wt = out["wav_predictions"][:, 0]
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    loudness.meter(wt, 16000, [len(x) for x in xs])
    assert _abi.launch_count() == n0 + 4
    n0 = _abi.launch_count()
    model.meter(out, 48000, loudness=-23, true_peak=-1)
    assert _abi.launch_count() == n0 + 11 + 4                 # the chain's loudness + true peak shape, then ev_meter
    n0 = _abi.launch_count()
    bad = [dict(sample_rate=11025), dict(sample_rate=16005), dict(sample_rate=192010), dict(lengths=[1, 2]),
           dict(lengths=[-1, 0, 0]), dict(lengths=[0, 0, wt.shape[1] + 1]), dict(lengths=[1.5, 1, 1]), dict(series=1)]
    for kw in bad:
        args = dict(sample_rate=16000)
        args.update(kw)
        with pytest.raises(ValueError):
            loudness.meter(wt, **args)
    for w in (wt.double(), wt.cpu(), wt[0], wt.half()):
        with pytest.raises(ValueError):
            loudness.meter(w, 16000)
    for kw in (dict(sample_rate=11025), dict(sample_rate=22050, loudness=1.0), dict(true_peak=3.0), dict(items=[5]),
               dict(watermark=0), dict(sample_rate=16001)):
        with pytest.raises(ValueError):
            model.meter(out, **kw)
    assert _abi.launch_count() == n0
    # the C entry point refuses bad arguments without launching
    starts = torch.tensor([0, wt.stride(0)], dtype=torch.int64, device=dev)
    n = torch.tensor([1000, 16000], dtype=torch.int64, device=dev)
    nh = np.array([1000, 16000], np.int64)
    kc = audio.k_weighting(16000)
    bank = torch.from_numpy(audio.limit_bank(16000, 16000)[0]).to(dev)
    res = torch.empty((6, 2), dtype=torch.float32, device=dev)
    ser = torch.empty((2, 2, 20), dtype=torch.float32, device=dev)
    nb = lib.ev_meter_workspace_bytes(2, 16000, 16000)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def call(wp=wt.data_ptr(), sp=starts.data_ptr(), k=2, sr=16000, bp=bank.data_ptr(), phases=bank.shape[0], taps=bank.shape[1],
             stride=20, wsb=nb, nhp=nh.ctypes.data):
        return lib.ev_meter(wp, sp, n.data_ptr(), nhp, k, sr, kc.ctypes.data, bp, phases, taps, res.data_ptr(), ser[0].data_ptr(),
                            ser[1].data_ptr(), stride, ws.data_ptr(), wsb, st)

    for kw in (dict(wp=None), dict(sp=None), dict(nhp=None), dict(k=0), dict(k=65536), dict(sr=11025), dict(sr=3990), dict(bp=None),
               dict(phases=65), dict(taps=20), dict(stride=9), dict(wsb=nb - 1)):
        assert call(**kw) == -1, kw
    assert lib.ev_meter_workspace_bytes(2, 16000, 11025) == 0 and lib.ev_meter_workspace_bytes(0, 16000, 16000) == 0
    assert _abi.launch_count() == n0
    assert call() == 0 and call(bp=None, phases=0) == 0
    assert _abi.launch_count() == n0 + 8
