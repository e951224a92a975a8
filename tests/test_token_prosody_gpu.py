"""Phoneme-level prosody controls and caller-given durations / pitch / energy on the GPU: the duration scan operator with
per-token scales bit for bit against torch, the whole path against the fixtures of the unmodified reference
(oracle/make_golden_token_prosody.py) in all four precision modes, the bitwise identities that need no oracle (predictions
fed back, constant rows, neutral tables, mixed batches, the front door), the launch count, and device-side errors."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import synth, _abi
from emotivoice_b200 import frontdoor as fd

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
EXTRA = ("duration_scale", "pitch_shift", "energy_scale", "durations", "pitch", "energy")
TOL = {"fp32": (1e-4, 1e-4), "fp32_ffma": (1e-4, 1e-4), "tf32": (5e-3, 2e-2), "bf16": (2e-2, 2e-2)}
ITEM_CASES = ["pause_word", "pitch_span", "caller_dur", "caller_pe", "mixed3"]
OUT_KEYS = ("dec_outputs", "wav_predictions", "log_duration_predictions", "pitch_predictions", "energy_predictions", "mel_lengths")


def extras_of(g):
    return {k: g[k].numpy() for k in EXTRA if k in g}


def _run(model, dev, batch, **kw):
    out = model(**{k: batch[k].to(dev) for k in KEYS}, **kw)
    torch.cuda.synchronize()
    return out


class _Precision:
    def __init__(self, model, mode, literal=False):
        self.model, self.mode, self.literal = model, mode, literal

    def __enter__(self):
        self.model.precision = self.mode
        self.model.compat_padded_batch = self.literal

    def __exit__(self, *exc):
        self.model.precision = "fp32"
        self.model.compat_padded_batch = False


def _same(a, b, keys=OUT_KEYS):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


# ---- the duration scan operator -----------------------------------------------------------------------------------------

def _scan(lib, dev, dur, lens, alpha, invariant, caller=0, max_frames=(1 << 24) - 1):
    """ev_op_duration_scan_controls with a (B,T) alpha (token stride 1) -> centers, ds, mel_lens, status (CPU)."""
    B, T = dur.shape
    centers, ds = torch.empty(B, T, device=dev), torch.empty(B, T, device=dev)
    mel = torch.empty(B + 1, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    dd, ld, ad = dur.to(dev), lens.to(torch.int32).to(dev), alpha.contiguous().to(dev)
    _abi.check(lib.ev_op_duration_scan_controls(dd.data_ptr(), caller, ld.data_ptr(), ad.data_ptr(), T, 1, invariant, B, T, max_frames,
                                                centers.data_ptr(), ds.data_ptr(), mel.data_ptr(), status.data_ptr(), None))
    torch.cuda.synchronize()
    return centers.cpu(), ds.cpu(), mel.cpu(), int(status.item())


def _torch_scan(dur, lens, alpha, invariant):
    """alignment.py:183-195 on the CPU with a (B,T) alpha: ds = d * alpha (fp32), the all-zero guard, cumsum - ds/2; frame counts
    trunc(fl32(exact sum))."""
    B, T = dur.shape
    centers, ds_out, n_exact = torch.zeros(B, T), torch.zeros(B, T), []
    if invariant:
        for b in range(B):
            tl = int(lens[b])
            ds = dur[b:b + 1, :tl] * alpha[b:b + 1, :tl]
            if ds.sum() == 0:
                ds[ds.sum(dim=1).eq(0)] = 1
            centers[b, :tl] = (ds.cumsum(dim=-1) - ds / 2)[0]
            ds_out[b, :tl] = ds[0]
            n_exact.append(int(np.float32(ds.double().sum().item())))
    else:
        ds = dur * alpha
        if ds.sum() == 0:
            ds[ds.sum(dim=1).eq(0)] = 1
        centers, ds_out = ds.cumsum(dim=-1) - ds / 2, ds
        n_exact = [int(np.float32(v)) for v in ds.double().sum(1).tolist()]
    return centers, ds_out, n_exact


@pytest.mark.parametrize("invariant", [1, 0], ids=["invariant", "literal"])
def test_per_token_scan_is_bitwise_torch(lib, dev, invariant):
    g = torch.Generator().manual_seed(11)
    n_items = 0
    for B, T in [(1, 1), (1, 31), (1, 33), (3, 100), (8, 257), (2, 1000), (5, 777)]:
        for draw in range(3):
            dur = torch.randint(0, 12, (B, T), generator=g)
            lens = torch.randint(1, T + 1, (B,), generator=g)
            lens[0] = T
            if B > 2:
                dur[1] = 0                                            # an all-zero item
            for b in range(B):
                dur[b, int(lens[b]):] = 0                             # pads are zero, as the predictor writes them
            lo, hi = [(1 / 16, 16.0), (0.5, 2.0), (0.9, 1.1)][draw]
            alpha = torch.exp(torch.rand(B, T, generator=g) * (np.log(hi) - np.log(lo)) + np.log(lo)).float()
            for zero_batch in ((False, True) if (B, T) == (3, 100) else (False,)):
                d = torch.zeros_like(dur) if zero_batch else dur
                for caller in (0, 1):
                    c, ds, mel, status = _scan(lib, dev, d, lens, alpha, invariant, caller)
                    c_ref, ds_ref, n_exact = _torch_scan(d, lens, alpha, invariant)
                    if invariant:
                        for b in range(B):
                            tl = int(lens[b])
                            assert torch.equal(c[b, :tl], c_ref[b, :tl]) and torch.equal(ds[b, :tl], ds_ref[b, :tl]), (B, T, b)
                    else:
                        assert torch.equal(c, c_ref) and torch.equal(ds, ds_ref), (B, T)
                    assert mel[:B].tolist() == n_exact and int(mel[B]) == max(n_exact), (B, T)
                    assert (status & 16) == 0
            n_items += B
    print("per-token duration scan: %d items bitwise" % n_items)


def test_per_item_strides_reproduce_the_existing_scan(lib, dev):
    """alpha item stride 1, token stride 0 through the new entry point == ev_op_duration_scan."""
    g = torch.Generator().manual_seed(5)
    dur = torch.randint(0, 9, (4, 300), generator=g)
    lens = torch.tensor([300, 120, 7, 299])
    for b in range(4):
        dur[b, int(lens[b]):] = 0
    al = (torch.rand(4, generator=g) * 3 + 0.2).float()
    B, T = dur.shape
    outs = []
    for new in (False, True):
        centers, ds = torch.empty(B, T, device=dev), torch.empty(B, T, device=dev)
        mel = torch.empty(B + 1, dtype=torch.int32, device=dev)
        dd, ld, ad = dur.to(dev), lens.to(torch.int32).to(dev), al.to(dev)
        if new:
            _abi.check(lib.ev_op_duration_scan_controls(dd.data_ptr(), 0, ld.data_ptr(), ad.data_ptr(), 1, 0, 1, B, T, (1 << 24) - 1,
                                                        centers.data_ptr(), ds.data_ptr(), mel.data_ptr(), None, None))
        else:
            _abi.check(lib.ev_op_duration_scan(dd.data_ptr(), ld.data_ptr(), ad.data_ptr(), 1, B, T, centers.data_ptr(), ds.data_ptr(),
                                               mel.data_ptr(), None))
        torch.cuda.synchronize()
        outs.append((centers.cpu(), ds.cpu(), mel.cpu()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def test_caller_scan_ignores_pads_and_flags_bad_durations(lib, dev):
    B, T = 3, 40
    lens = torch.tensor([40, 25, 10])
    alpha = torch.ones(B, T)
    dur = torch.randint(0, 6, (B, T), generator=torch.Generator().manual_seed(2))
    clean = dur.clone()
    for b in range(B):
        clean[b, int(lens[b]):] = 0
        dur[b, int(lens[b]):] = -7 if b == 1 else 10 ** 12      # garbage past the lengths: ignored, never flagged
    for invariant in (1, 0):
        got = _scan(lib, dev, dur, lens, alpha, invariant, caller=1)
        want = _scan(lib, dev, clean, lens, alpha, invariant, caller=1)
        for x, y in zip(got[:3], want[:3]):
            assert torch.equal(x, y)
        assert got[3] == 0
    # a negative duration: bit 16; the sums see it as 0, so the other items are untouched
    bad = clean.clone()
    bad[1, 3] = -5
    c, ds, mel, status = _scan(lib, dev, bad, lens, alpha, 1, caller=1)
    assert status & 16
    ok = clean.clone()
    ok[1, 3] = 0
    ref = _scan(lib, dev, ok, lens, alpha, 1, caller=1)
    assert mel.tolist() == ref[2].tolist()
    # an item whose frame count exceeds the limit, before or after scaling, sets bit 16
    for d0, a, limit in ((6000, 1.0, 5000), (1 << 40, 1.0, (1 << 23) - 1), (400, 16.0, 5000)):
        big = clean.clone()
        big[0, 0] = d0
        al = alpha.clone()
        al[0] = a
        assert _scan(lib, dev, big, lens, al, 1, caller=1, max_frames=limit)[3] & 16, (d0, a, limit)
    assert _scan(lib, dev, clean, lens, alpha, 1, caller=1, max_frames=int(clean.sum(1).max()))[3] == 0


# ---- the whole path against the reference fixtures ----------------------------------------------------------------------

@pytest.mark.parametrize("mode", list(TOL))
@pytest.mark.parametrize("name", ITEM_CASES)
def test_token_controls_match_reference_fixture(model, dev, name, mode):
    g = load_golden("token_prosody_" + name)
    tm, tw = TOL[mode]
    with _Precision(model, mode):
        out = _run(model, dev, g, **extras_of(g))
    T = out["log_duration_predictions"].shape[1]
    for b in range(g["inputs_ling"].shape[0]):
        n = int(g["input_lengths"][b])
        Fb = int(g["mel_lens_%d" % b][0])
        assert torch.equal(out["log_duration_predictions"][b, :n].cpu(), g["pred_durations_%d" % b][0])      # raw predictions
        assert int(out["mel_lengths"][b]) == Fb
        e_mel = rel_max(out["dec_outputs"][b, :Fb].cpu(), g["mel_%d" % b][0])
        e_wav = rel_rms(out["wav_predictions"][b, 0, :Fb * 256].cpu(), g["wav_%d" % b][0, 0])
        print(name, mode, b, "mel rel-max %.2e wav rel-rms %.2e" % (e_mel, e_wav))
        assert e_mel <= tm and e_wav <= tw
        assert rel_max(out["pitch_predictions"].reshape(-1, T)[b, :n].cpu(), g["pred_pitch_%d" % b][0]) <= 1e-4
        assert torch.count_nonzero(out["dec_outputs"][b, Fb:]) == 0


@pytest.mark.parametrize("mode", list(TOL))
def test_padded_literal_batch_with_token_controls(model, dev, mode):
    g = load_golden("token_prosody_padded")
    tm, tw = TOL[mode]
    with _Precision(model, mode, literal=True):
        out = _run(model, dev, g, **extras_of(g))
    assert torch.equal(out["log_duration_predictions"].cpu(), g["pred_durations"])
    assert out["mel_lengths"].cpu().tolist() == g["mel_lens"].tolist()
    assert out["dec_outputs"].shape == g["mel"].shape
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= tm
    assert rel_rms(out["wav_predictions"].cpu(), g["wav"]) <= tw


# ---- bitwise identities -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", list(TOL))
def test_predictions_fed_back_are_the_plain_forward(model, dev, mode):
    for name, literal in (("b1_t100", False), ("b3_padded", False), ("b3_padded", True)):
        g = load_golden(name)
        with _Precision(model, mode, literal):
            plain = _run(model, dev, g)
            fed = _run(model, dev, g, durations=plain["log_duration_predictions"], pitch=plain["pitch_predictions"],
                       energy=plain["energy_predictions"])
            host = _run(model, dev, g, durations=plain["log_duration_predictions"].cpu(), pitch=plain["pitch_predictions"].cpu())
        _same(fed, plain)
        _same(host, plain)


@pytest.mark.parametrize("mode", list(TOL))
def test_constant_rows_are_the_per_item_call_and_neutral_tables_no_call(model, dev, mode):
    g = load_golden("prosody_mixed3")
    c = {k: g[k].numpy() for k in ("duration_scale", "pitch_shift", "energy_scale")}
    T = int(g["inputs_ling"].shape[1])
    rows = {k: np.repeat(v[:, None], T, axis=1) for k, v in c.items()}
    with _Precision(model, mode):
        _same(_run(model, dev, g, **rows), _run(model, dev, g, **c))
        plain = _run(model, dev, g)
        _same(_run(model, dev, g, duration_scale=np.ones((3, T)), pitch_shift=torch.zeros(3, T), energy_scale=[[1.0] * T] * 3), plain)


@pytest.mark.parametrize("mode", list(TOL))
def test_mixed_token_batch_is_bitwise_each_b1_call(model, dev, mode):
    for name in ("token_prosody_mixed3", "token_prosody_caller_dur"):
        g = load_golden(name)
        x = extras_of(g)
        with _Precision(model, mode):
            out = _run(model, dev, g, **x)
            for b in range(g["inputs_ling"].shape[0]):
                n = int(g["input_lengths"][b])
                kw = {k: (v[b:b + 1, :n] if v.ndim == 2 else v[b:b + 1]) for k, v in x.items()}
                single = _run(model, dev, synth.slice_batch(g, b), **kw)
                Fb = int(out["mel_lengths"][b])
                assert int(single["mel_lengths"][0]) == Fb
                assert torch.equal(single["dec_outputs"][0], out["dec_outputs"][b, :Fb]), (name, b)
                assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256]), (name, b)


def test_controlled_forward_launches_what_a_per_item_one_launches(model, dev):
    """Same frame counts (the decoder's and vocoder's launch plans follow them), three ways of asking for them."""
    g = load_golden("prosody_mixed3")
    per_item = dict(duration_scale=[0.8, 1.0, 1.25], pitch_shift=[1.0, 0.0, -1.0])
    T = int(g["inputs_ling"].shape[1])
    rows = {k: np.repeat(np.asarray(v)[:, None], T, axis=1) for k, v in per_item.items()}
    plain = _run(model, dev, g)
    counts = []
    for kw in (per_item, rows, dict(rows, durations=plain["log_duration_predictions"], pitch=plain["pitch_predictions"].cpu())):
        _run(model, dev, g, **kw)                     # warm: workspaces and tables at their sizes
        n0 = _abi.launch_count()
        _run(model, dev, g, **kw)
        counts.append(_abi.launch_count() - n0)
    assert counts[0] == counts[1] == counts[2], counts


def test_invalid_device_durations_raise_and_the_engine_keeps_serving(model, dev):
    ok = load_golden("b1_t12")
    fresh = _run(model, dev, ok)
    d = fresh["log_duration_predictions"].clone()
    d[0, 3] = -1
    with pytest.raises(ValueError, match="negative"):
        _run(model, dev, ok, durations=d)
    d[0, 3] = 1 << 40                                 # far more frames than the vocoder can index
    with pytest.raises(ValueError, match="index"):
        _run(model, dev, ok, durations=d)
    for kw in (dict(durations=fresh["log_duration_predictions"].to(torch.int32)), dict(pitch=fresh["pitch_predictions"].double()),
               dict(durations=-torch.ones(1, 12, dtype=torch.int64))):
        with pytest.raises(ValueError):               # wrong device dtype, or negative on the host: raised before any enqueue
            _run(model, dev, ok, **kw)
    after = _run(model, dev, ok)
    g = ok
    assert rel_max(after["dec_outputs"][0].cpu(), g["mel"][0]) <= 1e-4
    _same(after, fresh)
    zf = load_golden("token_prosody_zero_frames")
    with pytest.raises(RuntimeError, match="no frames"):
        _run(model, dev, zf, **extras_of(zf))
    _same(_run(model, dev, ok), fresh)


def test_microbatcher_token_requests_are_each_the_b1_result(model, dev):
    g = load_golden("b3_padded")
    n = [int(v) for v in g["input_lengths"]]
    reqs = [dict(speed=[1.0 + 0.25 * (t % 3) for t in range(n[0])]), dict(speed=0.8, pitch_shift=[2.0] * n[1]), dict()]
    with fd.MicroBatcher(model, device=dev, max_batch=3, max_wait_s=0.5) as mb:
        futs = [mb.submit(g["inputs_ling"][b, :n[b]].numpy(), int(g["inputs_speaker"][b]), g["inputs_style_embedding"][b].numpy(),
                          g["inputs_content_embedding"][b].numpy(), **reqs[b]) for b in range(3)]
        outs = [f.result(timeout=120) for f in futs]
    assert mb.batches_run == 1
    for b in range(3):
        c = fd.phoneme_controls(n[b], **reqs[b])
        kw = {k: ([v] if np.ndim(v) == 0 else np.asarray(v)[None, :])
              for k, v in zip(("duration_scale", "pitch_shift", "energy_scale"), c)}
        single = _run(model, dev, synth.slice_batch(g, b), **kw)
        assert torch.equal(outs[b], single["wav_predictions"][0, 0].cpu()), b
    # caller durations through the front door, edited from a first synthesis
    one = synth.slice_batch(g, 1)
    first = _run(model, dev, one)
    d = first["log_duration_predictions"][0].cpu().numpy().copy()
    d[2] += 5
    with fd.MicroBatcher(model, device=dev, max_batch=2, max_wait_s=0.5) as mb:
        w = mb.submit(one["inputs_ling"][0].numpy(), int(one["inputs_speaker"][0]), one["inputs_style_embedding"][0].numpy(),
                      one["inputs_content_embedding"][0].numpy(), durations=d).result(timeout=120)
    single = _run(model, dev, one, durations=d[None, :])
    assert torch.equal(w, single["wav_predictions"][0, 0].cpu())
    assert int(single["mel_lengths"][0]) == int(first["mel_lengths"][0]) + 5
