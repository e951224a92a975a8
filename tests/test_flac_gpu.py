"""FLAC output on the GPU (``format_audio(encoding="flac")``, ``fetch_audio``, the MicroBatcher, ev_flac_encode): the file
images equal the numpy oracle's byte for byte, and decode to exactly the PCM16 ``fetch_audio`` returns, on the engine's outputs
(fixture utterances, a padded batch, a joined paragraph) at several rates with and without loudness normalisation, and on int16
items fed straight to the ABI (signals, block edges, one-sample items, a two-minute item); batch and order independence,
EV_PDL=0, argument errors, and a third-party decoder when one is installed."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from audio_cases import SR, engine_outputs
from conftest import ROOT
from emotivoice_b200 import _abi, synth
from emotivoice_b200 import frontdoor as fd
from oracle import flac_oracle as F
from test_flac import signals

pytestmark = pytest.mark.gpu
RATES = [8000, 16000, 24000, 44100, 48000, 127625]


def abi_flac(lib, dev, items, rate):
    """int16 items through ev_flac_encode -> list of bytes."""
    counts = np.array([len(x) for x in items], np.int64)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    pcm = torch.from_numpy(np.concatenate(items).astype(np.int16)).to(dev)
    pcm_off = torch.from_numpy(offs).to(dev)
    bound = sum(int(lib.ev_flac_bound_bytes(int(n))) for n in counts)
    out = torch.full((bound,), 0xA5, dtype=torch.uint8, device=dev)
    out_off = torch.empty(len(items) + 1, dtype=torch.int64, device=dev)
    nb = lib.ev_flac_workspace_bytes(len(items), int(counts.max()))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_flac_encode(pcm.data_ptr(), pcm_off.data_ptr(), len(items), counts.ctypes.data, rate, out.data_ptr(), bound,
                                  out_off.data_ptr(), ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    o = out_off.cpu().numpy()
    b = out.cpu().numpy().tobytes()
    return [b[o[k]:o[k + 1]] for k in range(len(items))]


def _check(img, pcm, rate, what):
    want = F.encode(pcm, rate)
    assert img == want, (what, len(img), len(want), next((i for i, (a, b) in enumerate(zip(img, want)) if a != b), None))
    r, y, _ = F.decode(img)
    assert r == rate and np.array_equal(y, pcm), what


@pytest.mark.parametrize("loudness", [None, -16.0])
@pytest.mark.parametrize("rate", RATES)
def test_engine_outputs_equal_the_oracle(model, dev, rate, loudness):
    for name, (out, _) in engine_outputs(model, dev).items():
        imgs = fd.fetch_audio(model, out, rate, "flac", loudness=loudness)
        pcms = fd.fetch_audio(model, out, rate, "pcm16", loudness=loudness)
        assert len(imgs) == len(pcms)
        for b, (img, pcm) in enumerate(zip(imgs, pcms)):
            assert img.dtype == np.uint8 and img.ndim == 1
            _check(img.tobytes(), pcm, rate, (name, b, rate, loudness))
        packed, offs = model.format_audio(out, rate, "flac", loudness=loudness)
        assert packed.dtype == torch.uint8 and packed.device == dev and offs.dtype == np.int64
        assert packed.numel() == offs[-1] and np.array_equal(np.diff(offs), [len(i) for i in imgs])
        if rate == SR and loudness is None:
            print(name, "flac / pcm16 bytes:", [round(len(i) / (2 * len(p)), 3) for i, p in zip(imgs, pcms)])


def direct_items():
    """int16 items for the ABI: the test signals, lengths on block edges, one-sample items."""
    sig = signals(n=2 * 4096 + 777, seed=5)
    rng = np.random.default_rng(11)
    items = dict(sig)
    for n in (1, 2, 12, 13, 255, 256, 257, 4095, 4096, 4097, 8191, 8192, 8193):
        items["noise_%d" % n] = np.clip(np.round(rng.normal(0, 2000, n) + 3000 * np.sin(np.arange(n) * 0.02)), -32768, 32767).astype(np.int16)
    items["one_max"] = np.array([32767], np.int16)
    items["one_min"] = np.array([-32768], np.int16)
    items["one_zero"] = np.array([0], np.int16)
    return items


@pytest.mark.parametrize("rate", [16000, 44100, 127625])
def test_direct_items_equal_the_oracle_in_any_batch_and_order(lib, dev, rate):
    items = direct_items()
    names, xs = list(items), list(items.values())
    batch = abi_flac(lib, dev, xs, rate)
    rev = abi_flac(lib, dev, xs[::-1], rate)[::-1]
    kinds = set()
    for name, x, img, r in zip(names, xs, batch, rev):
        _check(img, x, rate, name)
        assert r == img, name
        assert abi_flac(lib, dev, [x], rate)[0] == img, name
        kinds |= {s["type"] for s in F.decode(img)[2]}
    assert kinds == {"CONSTANT", "FIXED", "LPC", "VERBATIM"}


def test_two_minute_item(lib, dev):
    n = 120 * SR + 1234
    t = np.arange(n)
    rng = np.random.default_rng(120)
    env = 0.5 + 0.5 * np.sin(2 * np.pi * t / (SR * 7.3))
    x = np.clip(np.round(env * (6000 * np.sin(2 * np.pi * 180 * t / SR) + 2500 * np.sin(2 * np.pi * 1210 * t / SR))
                         + rng.normal(0, 60, n)), -32768, 32767).astype(np.int16)
    img = abi_flac(lib, dev, [np.zeros(5, np.int16), x], SR)[1]
    _check(img, x, SR, "two_minutes")
    print("two-minute item: %d bytes, %.3f of PCM16" % (len(img), len(img) / (2 * n)))


def pdl_dump(path):
    """FLAC images of the direct items through the ABI (run under EV_PDL=0 by the test below)."""
    from emotivoice_b200 import build
    build.build(verbose=False)
    lib = _abi.load()
    imgs = abi_flac(lib, torch.device("cuda:0"), list(direct_items().values()), 24000)
    np.savez(path, *[np.frombuffer(b, np.uint8) for b in imgs])


def test_same_bytes_with_pdl_off(tmp_path):
    here = str(tmp_path / "pdl_on.npz")
    pdl_dump(here)
    off = str(tmp_path / "pdl_off.npz")
    path = [ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])
    env = dict(os.environ, EV_PDL="0", PYTHONPATH=os.pathsep.join(path))
    subprocess.run([sys.executable, "-c", "import test_flac_gpu as T, sys; T.pdl_dump(sys.argv[1])", off], env=env, check=True,
                   cwd=ROOT, timeout=600)
    x, y = np.load(here), np.load(off)
    assert x.files == y.files
    for k in x.files:
        assert np.array_equal(x[k], y[k]), k


def test_invalid_arguments(model, lib, dev):
    out, _ = engine_outputs(model, dev)["b3_padded"]
    torch.cuda.synchronize()
    n0 = _abi.launch_count()
    for kw in (dict(sample_rate=3999), dict(sample_rate=44100.5), dict(items=[3]), dict(loudness=1.0), dict(encoding="FLAC")):
        args = dict(sample_rate=None, encoding="flac")
        args.update(kw)
        with pytest.raises(ValueError):
            model.format_audio(out, **args)
        with pytest.raises(ValueError):
            fd.fetch_audio(model, out, **args)
    assert _abi.launch_count() == n0
    xs = [np.arange(5000, dtype=np.int16), np.ones(3, np.int16)]
    counts = np.array([5000, 3], np.int64)
    pcm = torch.from_numpy(np.concatenate(xs)).to(dev)
    pcm_off = torch.tensor([0, 5000, 5003], dtype=torch.int64, device=dev)
    bound = sum(int(lib.ev_flac_bound_bytes(int(n))) for n in counts)
    o = torch.empty(bound, dtype=torch.uint8, device=dev)
    oo = torch.empty(3, dtype=torch.int64, device=dev)
    nb = lib.ev_flac_workspace_bytes(2, 5000)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    zero = np.array([5000, 0], np.int64)

    def call(p=pcm.data_ptr(), po=pcm_off.data_ptr(), n=2, c=counts.ctypes.data, rate=16000, out=o.data_ptr(), ob=bound,
             oop=oo.data_ptr(), w=ws.data_ptr(), wb=nb):
        return lib.ev_flac_encode(p, po, n, c, rate, out, ob, oop, w, wb, st)

    for kw in (dict(p=None), dict(po=None), dict(c=None), dict(out=None), dict(oop=None), dict(w=None), dict(n=0), dict(n=65536),
               dict(rate=3999), dict(rate=192001), dict(c=zero.ctypes.data), dict(ob=bound - 1), dict(wb=nb - 1)):
        rc = call(**kw)
        assert rc == -1, kw
        with pytest.raises(_abi.EvError):
            _abi.check(rc)
    assert lib.ev_flac_bound_bytes(0) == 0 and lib.ev_flac_workspace_bytes(0, 10) == 0 and lib.ev_flac_workspace_bytes(1, 0) == 0
    assert _abi.launch_count() == n0
    assert call() == 0
    assert _abi.launch_count() == n0 + 4


def test_microbatcher_flac_equals_fetch_audio_alone(model, dev):
    rng = np.random.default_rng(43)
    utts = [synth.make_utterance(rng, int(n)) for n in (14, 33, 9, 21)]
    fmts = [(None, "flac", None), (48000, "flac", -16.0), (8000, "mulaw", None), (None, "pcm16", None)]
    with fd.MicroBatcher(model, device=dev, max_batch=4, max_wait_s=0.5) as mb:
        futs = [mb.submit(u["ids"], int(u["speaker"]), u["style"], u["content"], sample_rate=r, encoding=e, loudness=t)
                for u, (r, e, t) in zip(utts, fmts)]
        got = [f.result(timeout=120) for f in futs]
        assert mb.batches_run <= 2
    for u, (r, e, t), w in zip(utts, fmts, got):
        single = model(**fd.collate([(u["ids"], int(u["speaker"]), u["style"], u["content"])], dev))
        want = fd.fetch_audio(model, single, r, e, loudness=t)[0]
        assert w.dtype == want.dtype and np.array_equal(w, want), (r, e, t)
        if e == "flac":
            assert np.array_equal(F.decode(w.tobytes())[1], fd.fetch_audio(model, single, r, "pcm16", loudness=t)[0])


def test_third_party_decoder_when_installed(model, dev, tmp_path):
    tool = shutil.which("flac") or shutil.which("ffmpeg")
    if tool is None:
        pytest.skip("no flac or ffmpeg binary on this machine")
    out, _ = engine_outputs(model, dev)["b1_t100"]
    img = fd.fetch_audio(model, out, 24000, "flac")[0]
    pcm = fd.fetch_audio(model, out, 24000, "pcm16")[0]
    src, dst = tmp_path / "a.flac", tmp_path / "a.raw"
    src.write_bytes(img.tobytes())
    if os.path.basename(tool) == "flac":
        cmd = [tool, "-d", "-s", "--force-raw-format", "--endian=little", "--sign=signed", "-o", str(dst), str(src)]
    else:
        cmd = [tool, "-v", "error", "-i", str(src), "-f", "s16le", "-acodec", "pcm_s16le", str(dst)]
    subprocess.run(cmd, check=True, timeout=120)
    assert np.array_equal(np.fromfile(dst, "<i2"), pcm)
