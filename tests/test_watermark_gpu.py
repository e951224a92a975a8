"""The watermark on the GPU (``format_audio(watermark=KEY)`` / ``ev_watermark_embed``, ``watermark.detect`` /
``ev_watermark_detect``): samples and statistics against the fp64 oracle, bitwise batch / order / EV_PDL=0 independence, the
unmarked chain unchanged, launch counts, detection in every output format after loudness and the limiter, crops, other keys,
noise and silence, and argument errors.

Tolerances.  The embed is fp32 FFTs of 1024 points: its change d is about 0.07 of the signal and carries fp32 relative error
near 1e-6, and y = x + d is rounded to fp32, so each sample is held to EMBED_TOL of its item's peak.  Detection is held to
Z_TOL: b sums up to 64 frames of ratios C / M, each with fp32 error near 1e-6 where M is well above the frame's rounding and more
where it is not (9.3e-4 was measured on the speech-like crop, 4e-6 on noise).

Detection.  A marked cell moves u = C / M by about alpha sin^2(phase), alpha / 2 on average, while u itself varies by about
1 / sqrt(2), so z grows as alpha sqrt(cells / 2), about 4.0 per sqrt(second) of a fully active band: 3 s of speech is not
enough.  An output is required to give z >= DETECT_Z when it holds at least MIN_S[rate] seconds, the shortest length at which
every seeded speech-like signal reached it (tools/watermark_timing.py; on an H100 80GB HBM3 at 700 W, though z does not
depend on the card): 5 s at 11.025 kHz and above, 15 s at 8 kHz G.711, whose quantisation noise buries the quieter cells of
the band.  The engine's outputs come from random weights and are not speech; they are held to the same lengths except at 8 kHz,
where they are only reported (6.2 and 6.5 were measured for the 8.6 s b1_t100 output)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audio_cases import SR, engine_outputs, out_dict, padded_batch
from conftest import ROOT
from emotivoice_b200 import _abi, watermark
from emotivoice_b200 import frontdoor as fd
from oracle import flac_oracle
from oracle import watermark_oracle as W
from test_watermark import speech_like

pytestmark = pytest.mark.gpu
KEY = 0x5EEDCAFEF00D
EMBED_TOL, Z_TOL = 1e-6, 1e-3
FORMATS = [(16000, "float32"), (16000, "pcm16"), (16000, "flac"), (8000, "mulaw"), (8000, "alaw"), (11025, "pcm16"),
           (22050, "pcm16"), (24000, "pcm16"), (44100, "pcm16"), (48000, "pcm16")]
CHAINS = [dict(), dict(loudness=-16.0), dict(loudness=-16.0, true_peak=-1.0)]
MIN_S = {8000: 12.0}                     # seconds; 5 s at every other rate
CROP_S = {16000: 6.0, 8000: 15.0}


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def abi_embed(lib, dev, w, lens, key=KEY, items=None):
    """ev_watermark_embed straight through the ABI -> host (k, stride) float32 (NaN where nothing was written)."""
    wt = torch.from_numpy(w).to(dev) if isinstance(w, np.ndarray) else w
    n_in = torch.tensor(lens, dtype=torch.int64, device=dev)
    k = len(lens) if items is None else len(items)
    it = None if items is None else torch.tensor(items, dtype=torch.int64, device=dev)
    out = torch.full((k, wt.stride(0)), np.nan, dtype=torch.float32, device=dev)
    _abi.check(lib.ev_watermark_embed(wt.data_ptr(), wt.stride(0), n_in.data_ptr(), None if it is None else it.data_ptr(), k, SR,
                                      key, out.data_ptr(), out.stride(0), _stream(dev)))
    return out.cpu().numpy()


def abi_detect(lib, dev, w, lens, key=KEY):
    """ev_watermark_detect through the ABI -> (z, offset, phase, per-tau best z, per-tau best m0) host arrays."""
    wt = torch.from_numpy(np.ascontiguousarray(w)).to(dev)
    n = torch.tensor(lens, dtype=torch.int64, device=dev)
    B = len(lens)
    z = torch.empty(B, dtype=torch.float32, device=dev)
    off = torch.empty(B, dtype=torch.int32, device=dev)
    ph = torch.empty(B, dtype=torch.int32, device=dev)
    nb = lib.ev_watermark_detect_workspace_bytes(B)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_watermark_detect(wt.data_ptr(), wt.stride(0), n.data_ptr(), B, key, z.data_ptr(), off.data_ptr(), ph.data_ptr(),
                                       ws.data_ptr(), nb, _stream(dev)))
    zt = ws[:4 * B * 512].view(torch.float32).view(B, 512).cpu().numpy()
    mt = ws[4 * B * 512:].view(torch.int32).view(B, 512).cpu().numpy()
    return z.cpu().numpy(), off.cpu().numpy(), ph.cpu().numpy(), zt, mt


def signals():
    rng = np.random.default_rng(21)
    return {"speech": speech_like(2.0, 1), "noise": (0.05 * rng.standard_normal(21000)).astype(np.float32),
            "short": speech_like(0.3, 2)[:700], "silence": np.zeros(9000, np.float32), "one": np.full(1, 0.25, np.float32)}


def test_embed_matches_the_oracle(lib, dev):
    sig = signals()
    w, lens = padded_batch(list(sig.values()))
    y = abi_embed(lib, dev, w, lens)
    for k, (name, x) in enumerate(sig.items()):
        yo = W.embed(x.astype(np.float64), KEY)
        peak = max(float(np.max(np.abs(yo))), 1e-30)
        err = float(np.max(np.abs(y[k, :len(x)] - yo)))
        print("embed %s: max |y - oracle| = %.3g (%.3g of peak %.3g)" % (name, err, err / peak, peak))
        assert err <= EMBED_TOL * peak, (name, err, peak)
        assert np.all(np.isnan(y[k, len(x):])), name                    # nothing past the item is written
    assert np.array_equal(y[3, :lens[3]], np.zeros(lens[3], np.float32))  # silence stays exactly silent
    d = y[0, :lens[0]].astype(np.float64) - sig["speech"]
    C, _ = W.mclt(sig["speech"].astype(np.float64), 0, np.arange(512))
    D, _ = W.mclt(d, 0, np.arange(512))
    D, C = D[1:-1], C[1:-1]                  # the first and last frames also see the item's edges
    out_band = np.r_[0:W.K_LO, W.K_HI:512]
    assert np.sum(D[:, out_band] ** 2) <= 1e-6 * np.sum(D ** 2)          # outside the band: only fp32 rounding of y
    ratio = 10 * np.log10(np.sum(D[:, W.K_LO:W.K_HI] ** 2) / np.sum(C[:, W.K_LO:W.K_HI] ** 2))
    print("mark / host in-band energy: %.2f dB" % ratio)
    assert abs(ratio + 20.0) < 1.0           # alpha^2 E[M^2] against E[C^2] = E[M^2] / 2


def test_detect_matches_the_oracle_at_every_grid(lib, dev):
    sig = {"speech": speech_like(0.5, 4), "noise": (0.1 * np.random.default_rng(3).standard_normal(6000)).astype(np.float32)}
    w, lens = padded_batch(list(sig.values()), poison=False)
    marked = abi_embed(lib, dev, w, lens)
    crop = [marked[0, 300:lens[0]], marked[1, :lens[1]], sig["noise"]]
    wc, lc = padded_batch(crop, poison=False)
    z, off, ph, zt, mt = abi_detect(lib, dev, wc[:, 0], lc)
    for k, x in enumerate(crop):
        zo, tau, m0, table = W.detect(x.astype(np.float64), KEY)
        best = table.max(axis=1)
        err = float(np.max(np.abs(zt[k] - best)))
        print("detect item %d: z %.4f (oracle %.4f) at (%d, %d) (oracle (%d, %d)); max per-tau error %.2g"
              % (k, z[k], zo, off[k], ph[k], tau, m0, err))
        assert err <= Z_TOL, (k, err)
        assert abs(z[k] - zo) <= Z_TOL and (off[k], ph[k]) == (tau, m0), k
        top2 = np.sort(table, axis=1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 2 * Z_TOL
        assert np.array_equal(mt[k][clear], table.argmax(axis=1)[clear]), k


def test_bitwise_in_any_batch_and_order(lib, dev):
    sig = signals()
    w, lens = padded_batch(list(sig.values()))
    y = abi_embed(lib, dev, w, lens)
    rev = abi_embed(lib, dev, w, lens, items=list(range(len(lens)))[::-1])
    for k, (name, x) in enumerate(sig.items()):
        one = abi_embed(lib, dev, x[None, None, :].copy(), [len(x)])
        assert np.array_equal(one[0, :len(x)].view(np.int32), y[k, :len(x)].view(np.int32)), name
        assert np.array_equal(rev[len(lens) - 1 - k, :len(x)].view(np.int32), y[k, :len(x)].view(np.int32)), name
    z, off, ph, _, _ = abi_detect(lib, dev, np.nan_to_num(y), lens)
    for k in range(len(lens)):
        z1, o1, p1, _, _ = abi_detect(lib, dev, np.nan_to_num(y[k:k + 1]), [lens[k]])
        assert z1[0].view(np.int32) == z[k].view(np.int32) and (o1[0], p1[0]) == (off[k], ph[k]), k


def pdl_dump(path):
    """Marked outputs and detector results of a seeded batch through the ABI (run under EV_PDL=0 by the test below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    lib = _abi.load()
    dev = torch.device("cuda:0")
    w, lens = padded_batch(list(signals().values()))
    y = abi_embed(lib, dev, w, lens)
    z, off, ph, _, _ = abi_detect(lib, dev, np.nan_to_num(y), lens)
    np.savez(path, y=np.nan_to_num(y), z=z, off=off, ph=ph)


def test_bitwise_equal_with_pdl_off(tmp_path):
    here = str(tmp_path / "pdl_on.npz")
    pdl_dump(here)
    off = str(tmp_path / "pdl_off.npz")
    path = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, EV_PDL="0", PYTHONPATH=os.pathsep.join(path))
    subprocess.run([sys.executable, "-c", "import test_watermark_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=600)
    x, y = np.load(here), np.load(off)
    for k in ("y", "z", "off", "ph"):
        assert np.array_equal(x[k].view(np.int32), y[k].view(np.int32)), k


def test_launches_one_more_per_chain_shape(model, dev):
    out, _ = engine_outputs(model, dev)["b3_padded"]
    for chain, n in ((dict(), 1), (dict(loudness=-16.0), 3), (dict(true_peak=-1.0), 4), (dict(loudness=-16.0, true_peak=-1.0), 11)):
        for enc, extra in (("pcm16", 0), ("flac", 4)):
            n0 = _abi.launch_count()
            model.format_audio(out, 24000, enc, **chain, watermark=KEY)
            assert _abi.launch_count() - n0 == n + extra + 1, (chain, enc)
    empty = out_dict(np.zeros((2, 1, 64), np.float32), [0, 0], dev)
    n0 = _abi.launch_count()
    packed, _ = model.format_audio(empty, 24000, "pcm16", hop=1, watermark=KEY)
    assert _abi.launch_count() == n0 and packed.numel() == 0


def test_marked_chain_is_the_chain_of_the_marked_waveform(model, lib, dev):
    """format_audio(watermark=K) equals format_audio of the embed's output (the mark is the first stage), and without a key
    the output is the unmarked chain's."""
    out, wavs = engine_outputs(model, dev)["b3_padded"]
    lens = [len(x) for x in wavs]
    w, _ = padded_batch(wavs)
    y = abi_embed(lib, dev, w, lens)
    mout = out_dict(np.nan_to_num(y)[:, None, :].copy(), lens, dev)
    for rate, enc in ((24000, "pcm16"), (8000, "mulaw"), (16000, "flac")):
        for chain in CHAINS:
            a = fd.fetch_audio(model, out, rate, enc, **chain, watermark=KEY)
            b = fd.fetch_audio(model, mout, rate, enc, hop=1, **chain)
            plain = fd.fetch_audio(model, out, rate, enc, **chain)
            again = fd.fetch_audio(model, out, rate, enc, **chain, watermark=None)
            for k in range(len(lens)):
                assert np.array_equal(a[k], b[k]), (rate, enc, chain, k)
                assert np.array_equal(plain[k], again[k]) and not np.array_equal(plain[k], a[k]), (rate, enc, chain, k)


def _decode(x, rate, enc):
    """fetch_audio's result -> float64 samples at ``rate``."""
    if enc == "float32":
        return x.astype(np.float64)
    if enc == "pcm16":
        return x.astype(np.float64) / 32768
    if enc == "flac":
        _, pcm = flac_oracle.decode(bytes(x))[:2]
        return np.asarray(pcm, np.float64) / 32768
    c = x.astype(np.int64)
    if enc == "mulaw":
        u = ~c & 0xFF
        t = (((u & 0x0F) << 3) + 0x84) << ((u >> 4) & 7)
        return np.where(u & 0x80, 0x84 - t, t - 0x84) / 32768
    a = c ^ 0x55
    seg = (a >> 4) & 7
    t = ((a & 0x0F) << 4) + np.where(seg == 0, 8, 0x108)
    t = np.where(seg > 1, t << np.maximum(seg - 1, 0), t)
    return np.where(a & 0x80, t, -t) / 32768


def _detect_host(xs, rate, key=KEY):
    w = np.zeros((len(xs), max(len(x) for x in xs)), np.float32)
    for k, x in enumerate(xs):
        w[k, :len(x)] = x
    z, off, ph = watermark.detect(torch.from_numpy(w).cuda(), rate, key, lengths=[len(x) for x in xs])
    return z.cpu().numpy(), off.cpu().numpy(), ph.cpu().numpy()


def _inputs(model, dev):
    """name -> (out dict, hop, [seconds of each output]): the engine's fixture outputs and seeded speech-like signals."""
    cases = {name: (o, None, [len(x) / SR for x in xs]) for name, (o, xs) in engine_outputs(model, dev).items()}
    sp = [speech_like(s, 100 + i) for i, s in enumerate((3.0, 4.5, 6.0, 8.0, 12.0, 16.0))]
    w, lens = padded_batch(sp, poison=False)
    cases["speech_like"] = (out_dict(w, lens, dev), 1, [n / SR for n in lens])
    return cases


@pytest.mark.parametrize("rate,enc", FORMATS)
def test_detected_in_every_format(model, dev, rate, enc):
    cases = _inputs(model, dev)
    for name, (out, hop, secs) in cases.items():
        for chain in CHAINS:
            marked = [_decode(x, rate, enc) for x in fd.fetch_audio(model, out, rate, enc, hop=hop, **chain, watermark=KEY)]
            plain = [_decode(x, rate, enc) for x in fd.fetch_audio(model, out, rate, enc, hop=hop, **chain)]
            zm, _, _ = _detect_host(marked, rate)
            zp, _, _ = _detect_host(plain, rate)
            print("%s %d %s %s: seconds %s marked z %s unmarked z %s" % (name, rate, enc, chain, np.round(secs, 2), np.round(zm, 2),
                                                                       np.round(zp, 2)))
            for k, s in enumerate(secs):
                if s >= MIN_S.get(rate, 5.0) and (name == "speech_like" or rate != 8000):
                    assert zm[k] >= watermark.DETECT_Z, (name, chain, k, s, zm[k])
                assert zp[k] < watermark.DETECT_Z, (name, chain, k, zp[k])


def test_other_keys_noise_and_silence_are_not_detected(model, dev):
    out, hop, secs = _inputs(model, dev)["speech_like"]
    marked = [_decode(x, SR, "pcm16") for x in fd.fetch_audio(model, out, SR, "pcm16", hop=hop, watermark=KEY)]
    keys = np.random.default_rng(9).integers(1, 2 ** 63 - 1, 200, dtype=np.int64)
    worst = max(float(_detect_host(marked, SR, int(k))[0].max()) for k in keys)
    print("largest z over 200 other keys: %.2f" % worst)
    assert worst < watermark.DETECT_Z
    rng = np.random.default_rng(10)
    noise = [0.1 * rng.standard_normal(int(s * SR)) for s in (3, 10, 30)]
    zn, _, _ = _detect_host(noise, SR)
    print("noise z %s" % np.round(zn, 2))
    assert np.all(zn < watermark.DETECT_Z)
    z, off, ph = _detect_host([np.zeros(5 * SR), np.zeros(1)], SR)
    assert np.array_equal(z, [0.0, 0.0]) and np.array_equal(off, [0, 0]) and np.array_equal(ph, [0, 0])


def test_crops_are_detected_at_their_alignment(model, dev):
    x = speech_like(30.0, 55)
    out = out_dict(x[None, None, :].copy(), [len(x)], dev)
    y = fd.fetch_audio(model, out, SR, "float32", hop=1, watermark=KEY)[0]
    n = int(CROP_S[16000] * SR)
    starts = np.random.default_rng(12).integers(0, len(y) - n, 12)
    z, off, ph = _detect_host([y[c:c + n] for c in starts], SR)
    for k, c in enumerate(starts):
        tau = (-int(c)) % W.H
        m0 = ((int(c) + tau) // W.H) % W.P
        print("crop at %d: z %.2f at (%d, %d), true (%d, %d)" % (c, z[k], off[k], ph[k], tau, m0))
        assert z[k] >= watermark.DETECT_Z and (off[k], ph[k]) == (tau, m0), (c, z[k])
    y8 = fd.fetch_audio(model, out, 8000, "mulaw", hop=1, watermark=KEY)[0]
    n8 = int(CROP_S[8000] * 8000)
    starts8 = np.random.default_rng(13).integers(0, len(y8) - n8, 12)
    z8, _, _ = _detect_host([_decode(y8[c:c + n8], 8000, "mulaw") for c in starts8], 8000)
    print("8 kHz mu-law crops: z %s" % np.round(z8, 2))
    assert np.all(z8 >= watermark.DETECT_Z)


def test_invalid_arguments_raise_before_anything_is_enqueued(model, lib, dev):
    out, _ = engine_outputs(model, dev)["b1_t100"]
    w = torch.zeros((2, 4000), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    for kw in (dict(watermark=True), dict(watermark=0), dict(watermark=2 ** 63), dict(watermark=1.5),
               dict(watermark=3, sample_rate=4000), dict(watermark=3, sample_rate=3000)):
        with pytest.raises(ValueError):
            model.format_audio(out, **kw)
    bad = [(w.cpu(), SR, 1, None), (w.double(), SR, 1, None), (w[0], SR, 1, None), (w, 4000, 1, None), (w, 44100.5, 1, None),
           (w, SR, True, None), (w, SR, 0, None), (w, SR, 1, [4000]), (w, SR, 1, [4001, 0]), (w, SR, 1, [-1, 5]),
           (w, SR, 1, torch.tensor([1, 2], device=dev)), (w[:, :0], SR, 1, None)]
    for args in bad:
        with pytest.raises(ValueError):
            watermark.detect(*args)
    n_in = torch.full((2,), 4000, dtype=torch.int64, device=dev)
    dst = torch.empty((2, 4000), dtype=torch.float32, device=dev)
    for rate, key, k, ostride in ((24000, 1, 2, 4000), (SR, 0, 2, 4000), (SR, 2 ** 63, 2, 4000), (SR, 1, 0, 4000), (SR, 1, 2, 3999)):
        with pytest.raises(_abi.EvError):
            _abi.check(lib.ev_watermark_embed(w.data_ptr(), 4000, n_in.data_ptr(), None, k, rate, key, dst.data_ptr(), ostride,
                                              _stream(dev)))
    ws = torch.empty(lib.ev_watermark_detect_workspace_bytes(2), dtype=torch.uint8, device=dev)
    z = torch.empty(2, dtype=torch.float32, device=dev)
    i32 = torch.empty(2, dtype=torch.int32, device=dev)
    for key, k, nb in ((0, 2, ws.numel()), (1, 0, ws.numel()), (1, 2, ws.numel() - 1)):
        with pytest.raises(_abi.EvError):
            _abi.check(lib.ev_watermark_detect(w.data_ptr(), 4000, n_in.data_ptr(), k, key, z.data_ptr(), i32.data_ptr(), i32.data_ptr(),
                                               ws.data_ptr(), nb, _stream(dev)))
    assert _abi.launch_count() == n0
