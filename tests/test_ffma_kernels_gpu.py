"""The "fp32_ffma" path's kernels against fp64, at the engine's layers, tile variants and item edges, and the path end to end.

Operator level (cases: tests/ffma_cases.py; references and bound: tests/voc_ref.py, tests/am_ref.py).  Every kernel is one fp32
FFMA chain per output, so every valid element must satisfy |y - y64| <= 2^-14 m (m = the sum of the magnitudes of the terms that
enter it) and each result 5e-5 of max|y64|.  Rows past each item are NaN on input and must come out as exact zeros.  Bitwise: each
item of a batch against its own batch-1 launch (often another variant of conv1d_tm_kernel); an in-place residual against a
separate one; conv_post_kernel against the granule-planar conv_post on the same values; the vocoder on a channels-first mel
(transpose_cf_to_tm_kernel) against the same mel time-major.  End to end: the fp64 oracle at b1_t50, batch invariance of b3_padded
and of an 8-item mixed-length batch, and the literal padded batch against its fixture, all in "fp32_ffma".

Largest err/m measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), tau = 2^-14:
    conv1d_tm  acoustic model: qkv 2^-21.2  wo 2^-21.8  ffn1 2^-21.7  ffn2 2^-21.4  cond.wx 2^-21.6  pred 2^-21.7  to_mel 2^-21.7
               vocoder: pre 2^-21.6  ups0-3 2^-21.1 .. 2^-21.4  c1 2^-21.0 (C 64) .. 2^-21.4  c2 2^-21.1 (C 128) .. 2^-21.9
               launcher limits 2^-21.9
    conv_post  2^-24.1
ffn2's 4608-product chain stays at 2^-21.4 of m, near the random-sign estimate and far from its 2^-11.8 worst case.  End to end
at b1_t50 against fp64: mel rel-max 1.2e-6, wav rms-rel 2.8e-7.  The operator cases ran 48 distinct (layer, batch variant,
batch-1 variant) pairs, all bitwise, covering the engine's 38.  The whole file took 22 s.
"""
import math

import pytest
import torch

import am_plans
import ffma_cases as FC
import voc_plans
import voc_ref
from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import synth

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
WORST = {}
PAIRS = set()
CONV = FC.conv_cases()


def _assert_row(kernel, row):
    print(row)
    assert row["rc"] == 0, row
    WORST[kernel] = max(WORST.get(kernel, 0.0), row["err_m"])
    assert row["finite"], row
    assert row["pad_zero"], row
    assert row["bound_ok"], ("err/m %.3g (tau %.3g), rel_max %.3g" % (row["err_m"], voc_ref.TAU[1], row["rel_max"]), row)
    for k, v in row.items():
        if k.startswith("bitwise"):
            assert v, (k, row)


@pytest.mark.parametrize("i", range(len(CONV)), ids=[c["name"] for c in CONV])
def test_conv1d_tm_against_fp64(lib, dev, i):
    c = CONV[i]
    row = FC.run_conv(lib, dev, c, 1000 * i + 7)
    for v1 in row.get("item_variants", []):
        PAIRS.add((c["layer"], ("conv1d_tm",) + tuple(row["variant"]), ("conv1d_tm",) + tuple(v1)))
    _assert_row("conv1d_tm " + c["family"] + ("" if c["family"] == "limit" else " " + c["layer"]), row)


def test_rows_a_over_the_limit_is_rejected_before_any_launch(lib, dev):
    """BM 256 + (3 - 1) * 65 = 386 rows: the smallest A tile over the 384-row limit (with K odd, rows_a is even)."""
    assert am_plans.conv1d_plan(lib, 1, 700, 32, 32, 3, 65) is None
    x = torch.zeros(1, 700, 32, device=dev)
    w = torch.zeros(3, 32, 32, device=dev)
    out = torch.full((1, 700, 32), float("nan"), device=dev)
    torch.cuda.synchronize()
    n0 = lib.ev_launch_count()
    rc = lib.ev_op_conv1d(x.data_ptr(), w.data_ptr(), None, 0, None, out.data_ptr(), 1, 700, 32, 32, 3, 65, None, 1, 0, 0.0, 0, 0, 1.0,
                          torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc != 0 and b"rows_a=386" in lib.ev_last_error()
    assert lib.ev_launch_count() == n0 and bool(out.isnan().all())


@pytest.mark.parametrize("i", range(len(FC.POST_CASES)), ids=[c["name"] for c in FC.POST_CASES])
def test_conv_post_against_fp64(lib, dev, i):
    _assert_row("conv_post", FC.run_post(lib, dev, FC.POST_CASES[i], 100 + i))


def test_zz_every_engine_variant_pair_ran_bitwise():
    """The batch / batch-1 pairs of variants the cases above ran (and found bitwise equal) include every pair the engine can
    produce for the corpus's batches on this device."""
    _, want = FC.engine_pairs(_lib())
    if not PAIRS:
        pytest.skip("the operator cases did not run in this session")
    missing = want - PAIRS
    print("variant pairs run: %d; engine pairs: %d" % (len(PAIRS), len(want)))
    assert not missing, sorted(missing)
    assert any(pb != p1 for _, pb, p1 in PAIRS)


def _lib():
    from emotivoice_b200 import _abi
    return _abi.load()


# ---- transpose_cf_to_tm ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 45, 1024])
def test_channels_first_mel_equals_time_major(model, dev, F):
    eng = model._engine()
    mel = synth.make_mel(2, F, seed=F).to(dev)                       # (B, 80, F): 32 x 32 tiles partial in both dimensions
    try:
        model.precision = "fp32_ffma"
        a = eng.vocode(mel, False, None)
        b = eng.vocode(mel.transpose(1, 2).contiguous(), True, None)
        torch.cuda.synchronize()
    finally:
        model.precision = "fp32"
    assert torch.isfinite(a).all()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- launch lists --------------------------------------------------------------------------------------------------------
AM_POINTS = [(1, (100,)), (3, (9, 23, 14)), (32, None)]
VOC_POINTS = [(1, (1024,)), (3, (900, 517, 1)), (8, (700, 1, 150, 37, 260, 9, 64, 129))]


@pytest.mark.parametrize("invariant", [1, 0], ids=["invariant", "literal"])
def test_am_launch_list_matches_the_engine(model, lib, dev, invariant):
    eng = model._engine()
    try:
        model.precision = "fp32_ffma"
        for B, lens in AM_POINTS:
            lens = list(lens) if lens is not None else synth.corpus_lengths(B)
            bt = {k: v.to(dev) for k, v in synth.make_batch(lens, seed=7 + B).items()}
            torch.cuda.synchronize()
            n0 = lib.ev_launch_count()
            r = eng.acoustic(bt["inputs_ling"], bt["input_lengths"], bt["inputs_speaker"], bt["inputs_style_embedding"],
                             bt["inputs_content_embedding"], invariant)
            n1 = lib.ev_launch_count()
            torch.cuda.synchronize()
            want = am_plans.engine_launches(lib, B, bt["inputs_ling"].shape[1], r["F"], "fp32_ffma", invariant)
            assert ("splitk_reduce",) not in want and not any(k[0] == "attention_tc" for k in want)
            assert n1 - n0 == len(want), (B, r["F"], invariant, n1 - n0, len(want))
    finally:
        model.precision = "fp32"


@pytest.mark.parametrize("time_major", [False, True], ids=["channels_first", "time_major"])
def test_voc_launch_list_matches_the_engine(model, lib, dev, time_major):
    eng = model._engine()
    try:
        model.precision = "fp32_ffma"
        for B, lens in VOC_POINTS:
            F = max(lens)
            mel = synth.make_mel(B, F, seed=31 * B + F).to(dev)
            if time_major:
                mel = mel.transpose(1, 2).contiguous()
            ml = torch.tensor(lens, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            n0 = lib.ev_launch_count()
            eng.vocode(mel, time_major, ml.data_ptr())
            n1 = lib.ev_launch_count()
            torch.cuda.synchronize()
            want = voc_plans.engine_launches(lib, B, F, am_plans.FFMA, time_major=time_major)
            assert (("transpose",) in want) == (not time_major)
            assert n1 - n0 == len(want), (B, F, time_major, n1 - n0, len(want))
    finally:
        model.precision = "fp32"


# ---- end to end --------------------------------------------------------------------------------------------------------------
def _forward(model, dev, batch):
    out = model(**{k: batch[k].to(dev) for k in KEYS})
    torch.cuda.synchronize()
    return out


def test_error_vs_fp64_oracle(model, dev, sd, conf):
    from oracle import jets_oracle as O
    g = load_golden("b1_t50")
    model.precision = "fp32_ffma"
    try:
        out = _forward(model, dev, g)
    finally:
        model.precision = "fp32"
    o64 = O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, dtype=torch.float64)
    assert torch.equal(out["log_duration_predictions"].cpu(), o64["log_duration_predictions"].to(torch.int64))
    e_mel = rel_max(out["dec_outputs"].cpu().double(), o64["dec_outputs"])
    e_wav = rel_rms(out["wav_predictions"].cpu().double(), o64["wav_predictions"])
    print("fp32_ffma vs fp64: mel rel-max %.2e wav rms-rel %.2e" % (e_mel, e_wav))
    assert e_mel <= 1e-4 and e_wav <= 1e-4


def _variants_differ(lib, B, lens, frames):
    """Does some convolution of the forward run another conv1d_tm variant for one item alone than in the batch?"""
    T, F = max(lens), max(frames)
    batch = am_plans.engine_launches(lib, B, T, F, "fp32_ffma", 1) + voc_plans.engine_launches(lib, B, F, am_plans.FFMA, time_major=True)
    for n, f in zip(lens, frames):
        one = am_plans.engine_launches(lib, 1, n, f, "fp32_ffma", 1) + voc_plans.engine_launches(lib, 1, f, am_plans.FFMA, time_major=True)
        if any(a != b for a, b in zip(batch, one)):
            return True
    return False


@pytest.mark.parametrize("which", ["b3_padded", "cfg3_mixed8"])
def test_batch_invariance(model, lib, dev, which):
    """Every item's durations, mel and waveform are bitwise its own batch-1 run's, with some layer on another variant."""
    g = load_golden("b3_padded") if which == "b3_padded" else synth.make_batch([200, 20, 57, 133, 96, 164, 31, 75], seed=4242)
    model.precision = "fp32_ffma"
    try:
        out = _forward(model, dev, g)
        lens = g["input_lengths"].tolist()
        ml = out["mel_lengths"].cpu().tolist()[:len(lens)]
        assert _variants_differ(lib, len(lens), lens, ml)
        for b, n in enumerate(lens):
            one = _forward(model, dev, synth.slice_batch(g, b))
            f = one["dec_outputs"].shape[1]
            assert f == ml[b]
            assert torch.equal(one["log_duration_predictions"][0], out["log_duration_predictions"][b, :n])
            assert torch.equal(one["dec_outputs"][0].view(torch.int32), out["dec_outputs"][b, :f].view(torch.int32))
            assert torch.equal(one["wav_predictions"][0, 0].view(torch.int32), out["wav_predictions"][b, 0, :f * 256].view(torch.int32))
            assert torch.count_nonzero(out["wav_predictions"][b, 0, f * 256:]) == 0
    finally:
        model.precision = "fp32"


def test_padded_batch_compat_matches_reference_fixture(model, dev):
    g = load_golden("b3_padded")
    model.precision = "fp32_ffma"
    model.compat_padded_batch = True
    try:
        out = _forward(model, dev, g)
    finally:
        model.compat_padded_batch = False
        model.precision = "fp32"
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert out["dec_outputs"].shape == g["mel"].shape
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= 1e-4
    assert rel_rms(out["wav_predictions"].cpu(), g["wav"]) <= 1e-4


def test_zz_largest_err_over_m():
    """Prints the largest err/m per kernel and layer kind of this session's cases."""
    print("largest err/m per kernel and layer:", {k: "%.3g (2^%.1f)" % (v, math.log2(v) if v > 0 else -math.inf) for k, v in sorted(WORST.items())})
