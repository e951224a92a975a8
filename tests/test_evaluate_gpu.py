"""The comparison of syntheses with recordings on the GPU (``evaluate.compare``, ev_eval_compare): through the ABI with crafted
log-mels and F0 at the grid edges (1 x 1, one row, one column, lengths around 32, 64, 1024 and 4096, all-equal frames where
only the tie rule decides) with the path bitwise the fp64 oracle's; NaN-poisoned padding, batch, order and EV_PDL=0
independence; ``compare`` end to end on seeded speech-like signals (itself, half the gain, a semitone up, 48 kHz input
against its own resampling and against scipy's); paths of batches whose longest synthesis and longest recording are in
different rows; no host sync; the engine's outputs against a slower reading of the same text; launch counts and argument
errors."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.signal import lfilter, resample_poly

from audio_cases import KEYS
from conftest import ROOT, load_golden
from emotivoice_b200 import _abi, evaluate, feats, recordings
from oracle import eval_oracle as O
from test_audio_format_gpu import _check_float32, _reference

pytestmark = pytest.mark.gpu
SR = 16000
REL = 1e-12


def _rel(a, b):
    if math.isnan(b):
        return 0.0 if math.isnan(a) else math.inf
    return abs(a - b) / max(abs(b), 1e-300) if a != b else 0.0


def crafted(N, M, seed, equal=False):
    """Log-mels (80, N), (80, M) and F0 tracks: the ref a time-warped, noisy copy of the syn, both partly unvoiced."""
    rng = np.random.default_rng(seed)
    if equal:
        a = np.full((80, N), -3.25, np.float32)
        b = np.full((80, M), -3.25, np.float32)
    else:
        a = rng.normal(-5.0, 2.0, size=(80, N)).astype(np.float32)
        idx = np.clip(np.round(np.linspace(0, N - 1, M) + rng.normal(0, 1.5, M)), 0, N - 1).astype(int)
        b = (a[:, idx] + rng.normal(0, 0.3, size=(80, M))).astype(np.float32)
    fa = np.where(rng.random(N) > 0.3, rng.uniform(70, 400, N), 0.0)
    fb = np.where(rng.random(M) > 0.3, rng.uniform(70, 400, M), 0.0)
    return a, fa, b, fb


def abi_compare(lib, dev, pairs, poison=True, with_path=True):
    """ev_eval_compare of [(mel_syn, f0_syn, mel_ref, f0_ref)] -> host dict of stats, counts and paths."""
    B = len(pairs)
    ns = [p[0].shape[1] for p in pairs]
    nr = [p[2].shape[1] for p in pairs]
    Fs, Fr = max(ns) + 3, max(nr) + 5
    fill = np.nan if poison else 0.0
    ms = np.full((B, 80, Fs), fill, np.float32)
    mr = np.full((B, 80, Fr), fill, np.float32)
    fs = np.full((B, Fs), fill)
    fr = np.full((B, Fr), fill)
    for b, (a, fa, c, fc) in enumerate(pairs):
        ms[b, :, :ns[b]], fs[b, :ns[b]] = a, fa
        mr[b, :, :nr[b]], fr[b, :nr[b]] = c, fc
    t = [torch.from_numpy(x).to(dev) for x in (ms, fs, mr, fr)]
    cnt = torch.tensor(ns + nr, dtype=torch.int32, device=dev)
    max_n, max_m = max(ns), max(nr)
    stats = torch.empty((3, B), dtype=torch.float64, device=dev)
    counts = torch.empty((2, B), dtype=torch.int32, device=dev)
    stride = max_n + max_m - 1
    path = torch.full((B, stride, 2), 7, dtype=torch.int32, device=dev)
    nb = lib.ev_eval_workspace_bytes(B, max_n, max_m)
    ws = torch.full((nb,), 0xff, dtype=torch.uint8, device=dev)
    table = torch.from_numpy(O.cos_table()).to(dev)
    _abi.check(lib.ev_eval_compare(t[0].data_ptr(), t[1].data_ptr(), Fs, cnt.data_ptr(), max_n, t[2].data_ptr(), t[3].data_ptr(), Fr,
                                   cnt.data_ptr() + 4 * B, max_m, B, table.data_ptr(), stats.data_ptr(), counts.data_ptr(),
                                   path.data_ptr() if with_path else None, stride, ws.data_ptr(), nb,
                                   torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    st, c, p = stats.cpu().numpy(), counts.cpu().numpy(), path.cpu().numpy()
    out = []
    for b in range(B):
        P = int(c[1, b])
        if with_path:
            assert (p[b, P:] == -1).all()
        out.append(dict(mcd=st[0, b], f0_rmse=st[1, b], vuv_error=st[2, b], voiced_pairs=int(c[0, b]), path_length=P,
                        path=p[b, :P] if with_path else None))
    return out


def check_pair(got, pair, name):
    want = O.compare(*pair)
    assert got["path_length"] == want["path_length"], name
    assert np.array_equal(got["path"], want["path"]), name
    assert got["voiced_pairs"] == want["voiced_pairs"], name
    for k in ("mcd", "f0_rmse", "vuv_error"):
        assert _rel(got[k], want[k]) <= REL, (name, k, got[k], want[k])
    return want


SHAPES = [(1, 1), (1, 37), (45, 1), (64, 64), (31, 33), (33, 31), (63, 65), (65, 64), (1023, 1025), (1025, 1000), (300, 4096),
          (4095, 4096), (4096, 4096), (4096, 1)]


@pytest.mark.parametrize("N,M", SHAPES)
def test_crafted_pairs_match_the_oracle(lib, dev, N, M):
    pair = crafted(N, M, N * 7 + M)
    got = abi_compare(lib, dev, [pair])[0]
    want = check_pair(got, pair, (N, M))
    assert max(N, M) <= got["path_length"] <= N + M - 1
    print("N=%d M=%d P=%d mcd %.6f (oracle %.6f)" % (N, M, got["path_length"], got["mcd"], want["mcd"]))


@pytest.mark.parametrize("N,M", [(1, 9), (9, 1), (50, 70), (70, 50), (200, 200)])
def test_all_equal_frames_follow_the_tie_rule(lib, dev, N, M):
    pair = crafted(N, M, 5, equal=True)
    got = abi_compare(lib, dev, [pair])[0]
    check_pair(got, pair, (N, M))
    assert got["mcd"] == 0.0
    # every d and D is 0: backtracking from (N-1, M-1) takes the diagonal while it exists, then the first row or column
    if N <= M:
        want = [(0, j) for j in range(M - N)] + [(i, M - N + i) for i in range(N)]
    else:
        want = [(i, 0) for i in range(N - M)] + [(N - M + j, j) for j in range(M)]
    assert np.array_equal(got["path"], np.array(want, np.int32))


def _mixed():
    shapes = [(40, 60), (1, 1), (700, 650), (129, 3), (64, 64), (500, 900)]
    return [crafted(n, m, 100 + i) for i, (n, m) in enumerate(shapes)]


def _bits(r):
    return (np.float64(r["mcd"]).view(np.int64), np.float64(r["f0_rmse"]).view(np.int64), np.float64(r["vuv_error"]).view(np.int64),
            r["voiced_pairs"], r["path_length"])


def test_batch_order_and_poison_do_not_change_any_bit(lib, dev):
    pairs = _mixed()
    batch = abi_compare(lib, dev, pairs)
    zeros = abi_compare(lib, dev, pairs, poison=False)
    rev = abi_compare(lib, dev, pairs[::-1])[::-1]
    nopath = abi_compare(lib, dev, pairs, with_path=False)
    for b, pair in enumerate(pairs):
        alone = abi_compare(lib, dev, [pair])[0]
        check_pair(alone, pair, b)
        for other in (batch[b], zeros[b], rev[b], nopath[b]):
            assert _bits(other) == _bits(alone), b
        for other in (batch[b], zeros[b], rev[b]):
            assert np.array_equal(other["path"], alone["path"]), b


def pdl_dump(path):
    """ev_eval_compare results of the mixed batch and compare() of speech-like pairs (run under EV_PDL=0 below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    dev = torch.device("cuda:0")
    lib = _abi.load()
    res = abi_compare(lib, dev, _mixed())
    out = {"abi_%d_%s" % (b, k): np.asarray(v) for b, r in enumerate(res) for k, v in r.items()}
    syn, ref, ls, lr = _speech_pair(dev)
    c = evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True)
    out.update({k: getattr(c, k).cpu().numpy() for k in c._fields})
    np.savez(path, **out)


def test_same_bits_with_pdl_off(tmp_path):
    here, off = str(tmp_path / "on.npz"), str(tmp_path / "off.npz")
    pdl_dump(here)
    py = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(py), EV_PDL="0")
    subprocess.run([sys.executable, "-c", "import test_evaluate_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=900)
    x, y = np.load(here), np.load(off)
    assert sorted(x.files) == sorted(y.files)
    for k in x.files:
        assert x[k].tobytes() == y[k].tobytes(), k


# ---- compare() end to end --------------------------------------------------------------------------------------------------
FORMANTS = ((730, 1090, 2440), (270, 2290, 3010), (530, 1840, 2480), (300, 870, 2240), (640, 1190, 2390))


def speech(seconds, seed, semitones=0.0, floor=1e-3):
    """A seeded speech-like signal at 16 kHz: phrases of voiced syllables (a harmonic source with F0 gliding in 90-220 Hz,
    scaled by 2^(semitones / 12), through three formant resonators) separated by pauses, over a white noise floor that keeps
    every mel band above the log's 1e-5 clamp."""
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    out = np.zeros(n)
    t = int(0.2 * SR)
    while t < n:
        for _ in range(rng.integers(2, 6)):
            m = int(rng.uniform(0.15, 0.3) * SR)
            f0 = np.linspace(rng.uniform(90, 220), rng.uniform(90, 220), m) * 2.0 ** (semitones / 12.0)
            ph = 2 * np.pi * np.cumsum(f0) / SR
            src = sum(np.sin(h * ph) / h * (h * f0 < 7000) for h in range(1, 70))
            y = src
            for f in FORMANTS[rng.integers(len(FORMANTS))]:
                r, w = np.exp(-np.pi * 90.0 / SR), 2 * np.pi * f / SR
                y = lfilter([1 - r], [1, -2 * r * np.cos(w), r * r], y)
            seg = y * np.sin(np.pi * np.arange(m) / m) ** 0.5
            end = min(n, t + m)
            out[t:end] = seg[:end - t]
            t = end
            if t >= n:
                break
        t += int(rng.uniform(0.15, 0.4) * SR)
    out *= 0.5 / np.abs(out).max()
    out += floor * np.random.default_rng(seed + 1000).standard_normal(n)
    return out.astype(np.float32)


def _speech_pair(dev):
    syn = [speech(3.0, 1), speech(5.5, 2)]
    ref = [speech(3.2, 4, semitones=1.0), speech(5.5, 2) * np.float32(0.5)]
    return _rows(syn, dev), _rows(ref, dev), [len(x) for x in syn], [len(x) for x in ref]


def _rows(signals, dev):
    L = max(len(s) for s in signals) + 100
    w = np.full((len(signals), L), np.nan, np.float32)
    for b, s in enumerate(signals):
        w[b, :len(s)] = s
    return torch.from_numpy(w).to(dev)


def _host(c):
    return {k: (None if getattr(c, k) is None else getattr(c, k).cpu().numpy()) for k in c._fields}


def test_speech_against_itself_half_gain_and_a_semitone_up(dev):
    x = speech(6.0, 3)
    up = speech(6.0, 3, semitones=1.0)
    half = x * np.float32(0.5)
    w_syn = _rows([x, x, x], dev)
    w_ref = _rows([x, half, up], dev)
    n = [len(x)] * 3
    N = len(x) // 256 + 1
    floor = feats.stft_features(w_ref, 512, 256, feats.scipy_hann(dev), 0.0, bands=feats.mel_bands(SR, 80, 0.0, 8000.0, dev), lengths=n)[0]
    assert float(floor[1, :, :N].min()) > math.log(1e-5) + 1.0   # half the gain keeps every band clear of the clamp
    c = _host(evaluate.compare(w_syn, w_ref, syn_lengths=n, ref_lengths=n, return_path=True))
    print("itself: mcd %g vuv %g f0 %g" % (c["mcd"][0], c["vuv_error"][0], c["f0_rmse"][0]))
    print("x 0.5: mcd %.3g dB, vuv_error %.4f, f0_rmse %.3f cents over %d voiced pairs"
          % (c["mcd"][1], c["vuv_error"][1], c["f0_rmse"][1], c["voiced_pairs"][1]))
    print("semitone up: mcd %.3f dB, vuv_error %.4f, f0_rmse %.2f cents over %d voiced pairs, P %d"
          % (c["mcd"][2], c["vuv_error"][2], c["f0_rmse"][2], c["voiced_pairs"][2], c["path_length"][2]))
    assert c["mcd"][0] == 0.0 and c["vuv_error"][0] == 0.0 and c["f0_rmse"][0] == 0.0
    assert np.array_equal(c["path"][0, :N], np.stack([np.arange(N)] * 2, axis=1)) and c["path_length"][0] == N
    assert c["voiced_pairs"][0] > N // 3
    assert c["mcd"][1] < 0.01
    assert abs(c["f0_rmse"][2] - 100.0) <= 35.0


def test_gpu_features_fed_to_the_oracle_give_the_same_results(dev):
    syn, ref, ls, lr = _speech_pair(dev)
    c = _host(evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True))
    ms, fs = evaluate._features(syn.contiguous(), ls)
    mr, fr = evaluate._features(ref.contiguous(), lr)
    ms, fs, mr, fr = (t.cpu().numpy() for t in (ms, fs, mr, fr))
    for b in range(len(ls)):
        N, M = ls[b] // 256 + 1, lr[b] // 256 + 1
        want = O.compare(ms[b, :, :N], fs[b, :N], mr[b, :, :M], fr[b, :M])
        P = int(c["path_length"][b])
        assert P == want["path_length"] and np.array_equal(c["path"][b, :P], want["path"])
        assert int(c["voiced_pairs"][b]) == want["voiced_pairs"]
        for k in ("mcd", "f0_rmse", "vuv_error"):
            assert _rel(float(c[k][b]), want[k]) <= REL, (b, k)


def test_48k_input_gives_the_bits_of_its_16k_resampling(dev):
    xs = [resample_poly(speech(2.5, 7), 3, 1).astype(np.float32), resample_poly(speech(4.0, 8), 3, 1).astype(np.float32)]
    ys = [resample_poly(speech(2.7, 9), 3, 1).astype(np.float32), resample_poly(speech(4.0, 8, semitones=1.0), 3, 1).astype(np.float32)]
    s48, r48 = _rows(xs, dev), _rows(ys, dev)
    ls, lr = [len(x) for x in xs], [len(y) for y in ys]
    a = _host(evaluate.compare(s48, r48, sample_rate=48000, syn_lengths=ls, ref_lengths=lr, return_path=True))
    s16, ls16 = recordings.resample(s48.contiguous(), ls, 48000, SR)
    r16, lr16 = recordings.resample(r48.contiguous(), lr, 48000, SR)
    b = _host(evaluate.compare(s16, r16, syn_lengths=ls16, ref_lengths=lr16, return_path=True))
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_48k_input_against_scipy_resampling_to_16k(dev):
    """Independent of the resampler compare() uses: its 16 kHz input is within the resampler's tested bound of scipy's
    resample_poly in fp64, and compare() at 48 kHz agrees with compare() of that fp64 resampling rounded to fp32."""
    xs = [resample_poly(speech(3.0, 11), 3, 1).astype(np.float32), resample_poly(speech(4.5, 12), 3, 1).astype(np.float32)]
    ys = [resample_poly(speech(3.3, 13), 3, 1).astype(np.float32), resample_poly(speech(4.5, 12, semitones=1.0), 3, 1).astype(np.float32)]
    s48, r48 = _rows(xs, dev), _rows(ys, dev)
    ls, lr = [len(x) for x in xs], [len(y) for y in ys]
    for sig, t48, lens in ((xs, s48, ls), (ys, r48, lr)):
        got, lens16 = recordings.resample(t48.contiguous(), lens, 48000, SR)
        got = got.cpu().numpy()
        for b, x in enumerate(sig):
            y64, m = _reference(x, 1, 3)
            assert lens16[b] == len(y64)
            _check_float32(got[b, :lens16[b]], y64, m)
    a = _host(evaluate.compare(s48, r48, sample_rate=48000, syn_lengths=ls, ref_lengths=lr))
    s16 = [_reference(x, 1, 3)[0].astype(np.float32) for x in xs]
    r16 = [_reference(y, 1, 3)[0].astype(np.float32) for y in ys]
    b = _host(evaluate.compare(_rows(s16, dev), _rows(r16, dev), syn_lengths=[len(x) for x in s16], ref_lengths=[len(y) for y in r16]))
    for i in range(len(xs)):
        P = int(b["path_length"][i])
        print("48 kHz vs scipy 16 kHz, pair %d: mcd %.6f / %.6f dB, f0_rmse %.3f / %.3f cents, vuv_error %.4f / %.4f, P %d / %d"
              % (i, a["mcd"][i], b["mcd"][i], a["f0_rmse"][i], b["f0_rmse"][i], a["vuv_error"][i], b["vuv_error"][i],
                 a["path_length"][i], P))
        assert abs(a["mcd"][i] - b["mcd"][i]) <= 0.01
        assert abs(a["f0_rmse"][i] - b["f0_rmse"][i]) <= 2.0
        assert abs(a["vuv_error"][i] - b["vuv_error"][i]) <= 3.0 / P
        assert abs(int(a["path_length"][i]) - P) <= 3


def test_paths_when_the_longest_syn_and_ref_are_in_different_rows(dev):
    syn = [speech(1.0, 21), speech(4.0, 22), speech(2.0, 23)]
    ref = [speech(4.2, 24), speech(0.8, 25), speech(2.1, 26)]
    ls, lr = [len(x) for x in syn], [len(y) for y in ref]
    ws, wr = _rows(syn, dev), _rows(ref, dev)
    c = _host(evaluate.compare(ws, wr, syn_lengths=ls, ref_lengths=lr, return_path=True))
    ns, nr = [n // 256 + 1 for n in ls], [n // 256 + 1 for n in lr]
    assert c["path"].shape == (3, max(ns) + max(nr) - 1, 2)
    ms, fs = (t.cpu().numpy() for t in evaluate._features(ws, ls))
    mr, fr = (t.cpu().numpy() for t in evaluate._features(wr, lr))
    for b in range(3):
        want = O.compare(ms[b, :, :ns[b]], fs[b, :ns[b]], mr[b, :, :nr[b]], fr[b, :nr[b]])
        P = int(c["path_length"][b])
        assert P == want["path_length"] and np.array_equal(c["path"][b, :P], want["path"]), b
        assert (c["path"][b, P:] == -1).all(), b
        assert _rel(float(c["mcd"][b]), want["mcd"]) <= REL, b
        alone = _host(evaluate.compare(ws[b:b + 1], wr[b:b + 1], syn_lengths=ls[b:b + 1], ref_lengths=lr[b:b + 1], return_path=True))
        for k in ("mcd", "f0_rmse", "vuv_error", "voiced_pairs", "path_length"):
            assert alone[k][0].tobytes() == c[k][b].tobytes(), (b, k)
        assert np.array_equal(alone["path"][0, :P], c["path"][b, :P]), b


def test_compare_does_not_wait_for_the_device(dev):
    syn, ref, ls, lr = _speech_pair(dev)
    xs = _rows([resample_poly(speech(2.0, 31), 3, 1).astype(np.float32)], dev)
    calls = (lambda: evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True),
             lambda: evaluate.compare(xs, xs, sample_rate=48000))
    for f in calls:                               # the first call on a device builds its tables
        f()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for f in calls:
            f()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_engine_outputs_against_a_slower_reading(model, dev):
    g = load_golden("b3_padded")
    out = model(**{k: g[k].to(dev) for k in KEYS})
    syn = out["wav_predictions"][:, 0].clone()
    ls = [256 * int(n) for n in out["mel_lengths_host"]]
    slow = model(**{k: g[k].to(dev) for k in KEYS}, duration_scale=1.25)
    ref = slow["wav_predictions"][:, 0].clone()
    lr = [256 * int(n) for n in slow["mel_lengths_host"]]
    c = _host(evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True))
    for b in range(len(ls)):
        N, M = ls[b] // 256 + 1, lr[b] // 256 + 1
        P = int(c["path_length"][b])
        assert max(N, M) <= P <= N + M - 1
        path = c["path"][b, :P]
        assert tuple(path[0]) == (0, 0) and tuple(path[-1]) == (N - 1, M - 1)
        assert (np.diff(path, axis=0) >= 0).all() and (np.diff(path, axis=0).sum(axis=1) >= 1).all()
        print("engine item %d: N %d M %d P %d mcd %.3f dB vuv_error %.3f f0_rmse %.1f cents (%d voiced pairs)"
              % (b, N, M, P, c["mcd"][b], c["vuv_error"][b], c["f0_rmse"][b], c["voiced_pairs"][b]))


def test_launch_counts_and_argument_errors(lib, dev):
    syn, ref, ls, lr = _speech_pair(dev)
    evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr)                  # warm the caches
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    feats.stft_features(syn, 512, 256, feats.scipy_hann(dev), 0.0, bands=feats.mel_bands(SR, 80, 0.0, 8000.0, dev), lengths=ls)
    n_stft = _abi.launch_count() - n0
    n0 = _abi.launch_count()
    feats.pitch_track(syn, SR, 256, continuous=False, lengths=ls)
    n_pitch = _abi.launch_count() - n0
    n0 = _abi.launch_count()
    evaluate.compare(syn, ref, syn_lengths=ls, ref_lengths=lr, return_path=True)
    assert _abi.launch_count() == n0 + 2 * (n_stft + n_pitch) + 3
    n0 = _abi.launch_count()
    evaluate.compare(syn, ref, sample_rate=22050, syn_lengths=ls, ref_lengths=lr)
    assert _abi.launch_count() == n0 + 2 + 2 * (n_stft + n_pitch) + 3           # one ev_format_audio per side first
    n0 = _abi.launch_count()
    bad = [dict(sample_rate=3000), dict(sample_rate=16001), dict(syn_lengths=[640, ls[1]]), dict(ref_lengths=[lr[0]]),
           dict(ref_lengths=[lr[0], ref.shape[1] + 1]), dict(return_path="yes"), dict(sample_rate=48000, syn_lengths=[1920, ls[1]])]
    for kw in bad:
        with pytest.raises(ValueError):
            evaluate.compare(syn, ref, **kw)
    for s, r in ((syn.cpu(), ref), (syn.double(), ref), (syn, ref[:1]), (syn[0], ref), (syn, ref.half())):
        with pytest.raises(ValueError):
            evaluate.compare(s, r)
    long = torch.zeros((1, 4096 * 256), dtype=torch.float32, device=dev)
    with pytest.raises(ValueError):
        evaluate.compare(long, long)
    assert _abi.launch_count() == n0
    # the C entry point refuses bad arguments without launching
    m = torch.zeros((1, 80, 32), device=dev)
    f = torch.zeros((1, 32), dtype=torch.float64, device=dev)
    cnt = torch.tensor([20, 30], dtype=torch.int32, device=dev)
    table = torch.from_numpy(O.cos_table()).to(dev)
    st = torch.empty((3, 1), dtype=torch.float64, device=dev)
    co = torch.empty((2, 1), dtype=torch.int32, device=dev)
    pa = torch.empty((1, 49, 2), dtype=torch.int32, device=dev)
    nb = lib.ev_eval_workspace_bytes(1, 20, 30)
    ws = torch.empty((nb,), dtype=torch.uint8, device=dev)

    def call(mp=m.data_ptr(), k=1, max_n=20, max_m=30, frames=32, tp=table.data_ptr(), pp=pa.data_ptr(), stride=49, wsb=nb):
        return lib.ev_eval_compare(mp, f.data_ptr(), frames, cnt.data_ptr(), max_n, m.data_ptr(), f.data_ptr(), 32, cnt.data_ptr() + 4,
                                   max_m, k, tp, st.data_ptr(), co.data_ptr(), pp, stride, ws.data_ptr(), wsb,
                                   torch.cuda.current_stream(dev).cuda_stream)

    for kw in (dict(mp=None), dict(tp=None), dict(k=0), dict(k=65536), dict(max_n=0), dict(max_m=4097), dict(frames=19),
               dict(stride=48), dict(wsb=nb - 1)):
        assert call(**kw) == -1, kw
    assert lib.ev_eval_workspace_bytes(1, 4097, 30) == 0 and lib.ev_eval_workspace_bytes(0, 20, 30) == 0
    assert _abi.launch_count() == n0
    assert call() == 0 and call(pp=None, stride=0) == 0
    assert _abi.launch_count() == n0 + 6
