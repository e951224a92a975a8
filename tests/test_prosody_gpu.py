"""Prosody controls on the GPU: the duration scan operator bit for bit against torch, the whole path against the
fixtures of the unmodified reference (oracle/make_golden_prosody.py) in all four precision modes, neutral controls
bitwise equal to none, mixed-control batches bitwise equal to each item's B=1 call, the zero-frame error, a long
slowed-down utterance against the oracle, and the micro-batching front door."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import synth, _abi
from emotivoice_b200 import frontdoor as fd
from oracle import prosody_oracle as O

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
CONTROLS = ("duration_scale", "pitch_shift", "energy_scale")
# (mel rel-max, wav rel-rms) per precision mode: the bounds the uncontrolled path is held to
TOL = {"fp32": (1e-4, 1e-4), "fp32_ffma": (1e-4, 1e-4), "tf32": (5e-3, 2e-2), "bf16": (2e-2, 2e-2)}
ITEM_CASES = ["a050", "a080", "a125", "a200", "p_up4", "p_down4", "e070", "e130", "combined", "mixed3", "zero_dur"]


def controls_of(g):
    return {c: g[c].tolist() for c in CONTROLS}


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


# ---- the duration scan operator ----------------------------------------------------------------------------------------

def _torch_scan(dur, lens, alpha, invariant):
    """alignment.py:183-195 on the CPU: ds = d * alpha (fp32), the all-zero guard, cumsum - ds/2.  Frame counts:
    trunc(fl32(exact sum)); also returns torch.sum(ds).int(), which may differ within a few ulps of an integer."""
    B, T = dur.shape
    centers = torch.zeros(B, T)
    ds_out = torch.zeros(B, T)
    n_exact, n_torch = [], []
    if invariant:
        for b in range(B):
            tl = int(lens[b])
            ds = dur[b:b + 1, :tl] * float(alpha[b])
            if ds.sum() == 0:
                ds[ds.sum(dim=1).eq(0)] = 1
            centers[b, :tl] = (ds.cumsum(dim=-1) - ds / 2)[0]
            ds_out[b, :tl] = ds[0]
            n_exact.append(int(np.float32(ds.double().sum().item())))
            n_torch.append(int(torch.sum(ds, dim=-1).int()))
    else:
        ds = dur * alpha.reshape(B, 1)
        if ds.sum() == 0:
            ds[ds.sum(dim=1).eq(0)] = 1
        centers = ds.cumsum(dim=-1) - ds / 2
        ds_out = ds
        n_exact = [int(np.float32(v)) for v in ds.double().sum(1).tolist()]
        n_torch = torch.sum(ds, dim=-1).int().tolist()
    return centers, ds_out, n_exact, n_torch


@pytest.mark.parametrize("invariant", [1, 0], ids=["invariant", "literal"])
def test_duration_scan_is_bitwise_torch(lib, dev, invariant):
    g = torch.Generator().manual_seed(7)
    shapes = [(1, 1), (1, 31), (1, 32), (1, 33), (3, 100), (8, 257), (2, 1000), (5, 777)]
    alphas = [1.0, 0.5, 2.0, 0.25, 4.0, None]          # None: inexact, drawn per item
    n_cases = n_torch_diff = 0
    for B, T in shapes:
        for a in alphas:
            dur = torch.randint(0, 12, (B, T), generator=g)
            lens = torch.randint(1, T + 1, (B,), generator=g)
            lens[0] = T
            if B > 2:
                dur[1] = 0                                            # an all-zero item
            if invariant:
                for b in range(B):
                    dur[b, int(lens[b]):] = 0                         # pads are zero, as the predictor writes them
            al = (torch.rand(B, generator=g) * 5.95 + 0.05) if a is None else torch.full((B,), a)
            al = al.float()
            for zero_batch in ((False, True) if (B, T) == (3, 100) else (False,)):
                d = torch.zeros_like(dur) if zero_batch else dur
                centers = torch.empty(B, T, device=dev)
                ds = torch.empty(B, T, device=dev)
                mel = torch.empty(B + 1, dtype=torch.int32, device=dev)
                dd, ld, ad = d.to(dev), lens.to(torch.int32).to(dev), al.to(dev)
                _abi.check(lib.ev_op_duration_scan(dd.data_ptr(), ld.data_ptr() if invariant else None, ad.data_ptr(), invariant, B, T,
                                                   centers.data_ptr(), ds.data_ptr(), mel.data_ptr(), None))
                torch.cuda.synchronize()
                c_ref, ds_ref, n_exact, n_torch = _torch_scan(d, lens, al, invariant)
                centers, ds, mel = centers.cpu(), ds.cpu(), mel.cpu()
                if invariant:
                    for b in range(B):
                        tl = int(lens[b])
                        assert torch.equal(centers[b, :tl], c_ref[b, :tl]), (B, T, a, b)
                        assert torch.equal(ds[b, :tl], ds_ref[b, :tl]), (B, T, a, b)
                else:
                    assert torch.equal(centers, c_ref), (B, T, a)
                    assert torch.equal(ds, ds_ref), (B, T, a)
                assert mel[:B].tolist() == n_exact and int(mel[B]) == max(n_exact), (B, T, a)
                n_torch_diff += sum(int(x != y) for x, y in zip(n_exact, n_torch))
                n_cases += B
    print("duration scan: %d items bitwise; torch.sum(ds).int() differed by a frame on %d of them" % (n_cases, n_torch_diff))
    assert n_torch_diff <= max(1, n_cases // 100)


def test_duration_scan_without_alpha_is_the_integer_scan(lib, dev):
    """alpha NULL == alpha 1: the integer-duration results of the scan every existing caller relies on."""
    dur = torch.randint(0, 9, (4, 300), generator=torch.Generator().manual_seed(3))
    B, T = dur.shape
    outs = []
    for alpha in (None, torch.ones(B, device=dev)):
        centers, ds = torch.empty(B, T, device=dev), torch.empty(B, T, device=dev)
        mel = torch.empty(B + 1, dtype=torch.int32, device=dev)
        dd = dur.to(dev)
        _abi.check(lib.ev_op_duration_scan(dd.data_ptr(), None, None if alpha is None else alpha.data_ptr(), 0, B, T,
                                           centers.data_ptr(), ds.data_ptr(), mel.data_ptr(), None))
        torch.cuda.synchronize()
        outs.append((centers.cpu(), ds.cpu(), mel.cpu()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
    assert outs[0][2][:B].tolist() == dur.sum(1).tolist()
    assert torch.equal(outs[0][0], (dur.float().cumsum(-1) - dur.float() / 2))


# ---- the whole path against the reference fixtures --------------------------------------------------------------------

def _engine_sd(model, sd, g):
    if "dur_bias" in g:
        s = dict(sd)
        s["am.duration_predictor.linear.bias"] = torch.full_like(sd["am.duration_predictor.linear.bias"], float(g["dur_bias"]))
        model.load_state_dict(s)
    return model


@pytest.mark.parametrize("mode", list(TOL))
@pytest.mark.parametrize("name", ITEM_CASES)
def test_per_item_controls_match_reference_fixture(model, dev, sd, name, mode):
    g = load_golden("prosody_" + name)
    tm, tw = TOL[mode]
    _engine_sd(model, sd, g)
    try:
        with _Precision(model, mode):
            out = _run(model, dev, g, **controls_of(g))
    finally:
        if "dur_bias" in g:
            model.load_state_dict(sd)
    for b in range(g["inputs_ling"].shape[0]):
        n = int(g["input_lengths"][b])
        Fb = int(g["mel_lens_%d" % b][0])
        assert torch.equal(out["log_duration_predictions"][b, :n].cpu(), g["durations_%d" % b][0])
        assert int(out["mel_lengths"][b]) == Fb
        e_mel = rel_max(out["dec_outputs"][b, :Fb].cpu(), g["mel_%d" % b][0])
        e_wav = rel_rms(out["wav_predictions"][b, 0, :Fb * 256].cpu(), g["wav_%d" % b][0, 0])
        print(name, mode, b, "mel rel-max %.2e wav rel-rms %.2e" % (e_mel, e_wav))
        assert e_mel <= tm and e_wav <= tw
        assert rel_max(out["pitch_predictions"].reshape(-1, out["log_duration_predictions"].shape[1])[b, :n].cpu(),
                       g["pitch_%d" % b][0]) <= 1e-4                     # raw predictions
        assert torch.count_nonzero(out["dec_outputs"][b, Fb:]) == 0


@pytest.mark.parametrize("mode", list(TOL))
def test_padded_literal_batch_with_per_item_alpha(model, dev, mode):
    g = load_golden("prosody_padded")
    tm, tw = TOL[mode]
    with _Precision(model, mode, literal=True):
        out = _run(model, dev, g, **controls_of(g))
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert out["mel_lengths"].cpu().tolist() == g["mel_lens"].tolist()
    assert out["dec_outputs"].shape == g["mel"].shape
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= tm
    assert rel_rms(out["wav_predictions"].cpu(), g["wav"]) <= tw


@pytest.mark.parametrize("mode", list(TOL))
def test_neutral_controls_are_bitwise_no_controls(model, dev, mode):
    for name, literal in (("b1_t100", False), ("b3_padded", False), ("b3_padded", True)):
        g = load_golden(name)
        B = g["inputs_ling"].shape[0]
        with _Precision(model, mode, literal):
            ref = _run(model, dev, g)
            outs = [_run(model, dev, g, duration_scale=1.0, pitch_shift=0.0, energy_scale=1.0),
                    _run(model, dev, g, duration_scale=[1.0] * B, pitch_shift=torch.zeros(B), energy_scale=np.ones(B))]
        for o in outs:
            for k in ("dec_outputs", "wav_predictions", "log_duration_predictions", "pitch_predictions", "mel_lengths"):
                assert torch.equal(o[k], ref[k]), (name, literal, k)


@pytest.mark.parametrize("mode", list(TOL))
def test_mixed_controls_batch_is_bitwise_each_b1_call(model, dev, mode):
    g = load_golden("prosody_mixed3")
    c = controls_of(g)
    with _Precision(model, mode):
        out = _run(model, dev, g, **c)
        for b in range(3):
            kw = {k: v[b] for k, v in c.items()}
            single = _run(model, dev, synth.slice_batch(g, b), **kw)
            Fb = int(out["mel_lengths"][b])
            assert int(single["mel_lengths"][0]) == Fb
            assert torch.equal(single["dec_outputs"][0], out["dec_outputs"][b, :Fb])
            assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256])
            if kw == {"duration_scale": 1.0, "pitch_shift": 0.0, "energy_scale": 1.0}:      # the neutral item: no controls at all
                plain = _run(model, dev, synth.slice_batch(g, b))
                assert torch.equal(plain["wav_predictions"], single["wav_predictions"])


def test_zero_frame_item_raises_and_the_engine_keeps_serving(model, dev):
    g = load_golden("prosody_zero_frames")
    ok = load_golden("b1_t12")
    fresh = _run(model, dev, ok)
    with pytest.raises(RuntimeError, match="no frames"):
        _run(model, dev, g, **controls_of(g))
    both = {k: torch.cat([ok[k], g[k]]) for k in KEYS}          # same length (12): one batch, one item without frames
    with pytest.raises(RuntimeError, match="no frames"):
        _run(model, dev, both, duration_scale=[1.0, 0.01])
    after = _run(model, dev, ok)
    for k in ("dec_outputs", "wav_predictions", "mel_lengths"):
        assert torch.equal(after[k], fresh[k])
    # the literal padded batch only fails when the whole batch has no frames (F = 0), like the reference
    model.compat_padded_batch = True
    try:
        out = _run(model, dev, both, duration_scale=[1.0, 0.01])
        assert int(out["mel_lengths"][1]) == 0 and int(out["mel_lengths"][0]) == int(fresh["mel_lengths"][0])
    finally:
        model.compat_padded_batch = False


def test_slow_long_utterance_grows_tables_and_matches_oracle(model, dev, sd, conf):
    """duration_scale 4 (a serving speed of 0.25) on the 100-phoneme input: ~4x the frames, beyond the sizes the other
    tests have grown the workspaces and positional table to."""
    g = load_golden("b1_t100")
    out = _run(model, dev, g, duration_scale=4.0)
    o = O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, duration_scale=4.0)
    F = int(out["mel_lengths"][0])
    assert F == int(o["mel_lens"][0]) == 4 * int(g["mel"].shape[1]) and F > 2000
    assert torch.equal(out["log_duration_predictions"].cpu(), o["log_duration_predictions"])
    e_mel, e_wav = rel_max(out["dec_outputs"].cpu(), o["dec_outputs"]), rel_rms(out["wav_predictions"].cpu(), o["wav_predictions"])
    print("duration_scale 4: F=%d mel rel-max %.2e wav rel-rms %.2e" % (F, e_mel, e_wav))
    assert e_mel <= 1e-4 and e_wav <= 1e-4


def test_microbatcher_requests_with_different_speeds_are_each_the_b1_result(model, dev):
    g = load_golden("b3_padded")
    speeds = [1.0, 1.25, 0.8]
    with fd.MicroBatcher(model, device=dev, max_batch=3, max_wait_s=0.5) as mb:
        futs = [mb.submit(g["inputs_ling"][b, :int(g["input_lengths"][b])].numpy(), int(g["inputs_speaker"][b]),
                          g["inputs_style_embedding"][b].numpy(), g["inputs_content_embedding"][b].numpy(), speed=speeds[b])
                for b in range(3)]
        outs = [f.result(timeout=120) for f in futs]
    assert mb.batches_run == 1
    for b in range(3):
        single = _run(model, dev, synth.slice_batch(g, b), duration_scale=1.0 / speeds[b])
        assert torch.equal(outs[b], single["wav_predictions"][0, 0].cpu())
