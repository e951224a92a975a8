"""GPU tests written after the last hardware run of round 1 (the round's GPU budget was spent): the bf16 precision
mode per operator and its batch invariance (its end-to-end accuracy is in test_gp_gpu.py), and the micro-batching queue
on the real engine.  The file name sorts last on purpose: under `pytest -m gpu -x` a failure in a test that has never
run on a GPU must not hide the suite that has.  The bf16 forward itself was measured once (tools/quick_fwd.py bf16: durations identical, wav 8.8e-4);
the tolerances are <= 4x the CPU emulation of the mode (profiles/r01_precision_emulation_cpu.json).  Fold these back
into test_tc_gpu.py / test_e2e_gpu.py once they have run green on hardware."""
import pytest
import torch

from conftest import load_golden, rel_max
from emotivoice_b200 import synth
from test_tc_gpu import KEYS, TC_CASES, check_conv1d_tc_epilogue_and_ragged, check_conv1d_tc_matches_torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,L,Cin,Cout,K,dil", [c for c in TC_CASES if c[2] % 16 == 0])      # bf16: 16 channels per MMA K step
def test_conv1d_tc_bf16_matches_torch(lib, dev, B, L, Cin, Cout, K, dil):
    check_conv1d_tc_matches_torch(lib, dev, B, L, Cin, Cout, K, dil, 2)


def test_conv1d_tc_bf16_epilogue_and_ragged(lib, dev):
    check_conv1d_tc_epilogue_and_ragged(lib, dev, 2)


def test_bf16_mode_is_batch_invariant(model, dev):
    from emotivoice_b200 import synth
    g = load_golden("b3_padded")
    model.precision = "bf16"
    try:
        out = model(**{k: g[k].to(dev) for k in KEYS})
        for b in range(3):
            single = model(**{k: v.to(dev) for k, v in synth.slice_batch(g, b).items()})
            Fb = single["dec_outputs"].shape[1]
            assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256])
    finally:
        model.precision = "fp32"


def test_microbatcher_on_the_engine_equals_b1_calls(model, dev):
    """SURVEY.md s8f rank 3: concurrent requests grouped into one padded forward return exactly (bitwise) what a
    B=1 call returns for each of them."""
    import numpy as np
    from emotivoice_b200 import frontdoor as fd
    rng = np.random.default_rng(11)
    utts = [synth.make_utterance(rng, int(n)) for n in (14, 33, 9, 21)]
    with fd.MicroBatcher(model, device=dev, max_batch=4, max_wait_s=0.5) as mb:
        futs = [mb.submit(u["ids"], int(u["speaker"]), u["style"], u["content"]) for u in utts]
        got = [f.result(timeout=120) for f in futs]
        assert mb.batches_run <= 2
    for u, w in zip(utts, got):
        single = model(**fd.collate([(u["ids"], int(u["speaker"]), u["style"], u["content"])], dev))
        assert torch.equal(single["wav_predictions"][0, 0].cpu(), w)


def test_fetch_pcm16_trims_and_matches_the_callers_cast(model, dev):
    """SURVEY.md s8f rank 2: GPU int16 conversion + one pinned D2H + per-item trim == what the reference callers compute
    from the fp32 waveform on the host (inference_am_vocoder_joint.py:130-131: `wav * 32768` -> `.astype('int16')`)."""
    import numpy as np
    from emotivoice_b200 import frontdoor as fd
    g = load_golden("b3_padded")
    out = model(**{k: g[k].to(dev) for k in KEYS})
    got = fd.fetch_pcm16(model, out)
    wav, lens = out["wav_predictions"].cpu().numpy(), out["mel_lengths"].cpu().tolist()
    assert len(got) == 3
    for b in range(3):
        want = (wav[b, 0, :lens[b] * 256] * 32768.0).astype("int16")
        assert got[b].dtype == np.int16 and np.array_equal(got[b], want)


# ---- style encoder (SURVEY.md s8f rank 1): BERT forward on the engine's kernels ------------------------------------------

STYLE_KEYS = ("input_ids", "token_type_ids", "attention_mask")
STYLE_OUTS = ("pooled_output", "pitch_outputs", "speed_outputs", "energy_outputs", "emotion_outputs")
_style_models = {}


def _style_model(small, dev):
    """One StyleEncoder per size for the whole session (BERT-base: 110 M seeded weights, packed once)."""
    if small not in _style_models:
        from types import SimpleNamespace
        from emotivoice_b200.style import StyleEncoder
        sc = synth.style_config(small)
        conf = SimpleNamespace(bert_path="(offline)", bert_hidden_size=sc.hidden_size, style_dim=sc.style_dim,
                               pitch_n_labels=sc.pitch_n_labels, speed_n_labels=sc.speed_n_labels,
                               energy_n_labels=sc.energy_n_labels, emotion_n_labels=sc.emotion_n_labels)
        m = StyleEncoder(conf, bert_config=dict(sc), _init=synth.make_style_state_dict(sc)).to(dev).eval()
        _style_models[small] = m
    return _style_models[small]


@pytest.mark.parametrize("name,small", [("style_small_b3", True), ("style_small_b1_n40", True), ("style_base_b2", False)])
def test_style_encoder_matches_reference_fixture(lib, dev, name, small):
    """Fixtures come from the reference's StyleEncoder class driving transformers' BertModel (oracle/make_golden_style.py).
    Default mode is 3xTF32 (fp32-accurate): 1e-4 of max|ref| through 12 post-LN layers (the two fp32 CPU evaluation orders
    already differ by 4e-6); tf32 mode: 2e-2."""
    m = _style_model(small, dev)
    g = load_golden(name)
    out = m(**{k: g[k].to(dev) for k in STYLE_KEYS})
    torch.cuda.synchronize()
    assert list(out.keys()) == list(STYLE_OUTS)
    for k in STYLE_OUTS:
        err = rel_max(out[k].cpu(), g[k])
        print(name, k, "rel-max %.2e" % err)
        assert out[k].shape == g[k].shape and err <= 1e-4
    m.precision = "tf32"
    try:
        out = m(**{k: g[k].to(dev) for k in STYLE_KEYS})
        assert rel_max(out["pooled_output"].cpu(), g["pooled_output"]) <= 2e-2
    finally:
        m.precision = "fp32"


def test_style_encoder_padding_is_invisible_and_errors_are_loud(lib, dev):
    """A right-padded item equals the same item alone, bitwise (key mask + batch-invariant GEMM plans); malformed masks and
    out-of-range ids raise like the library the reference uses would (IndexError from the embedding lookup)."""
    m = _style_model(True, dev)
    g = load_golden("style_small_b3")
    full = m(**{k: g[k].to(dev) for k in STYLE_KEYS})
    for b in range(3):
        n = int(g["attention_mask"][b].sum())
        alone = m(**{k: g[k][b:b + 1, :n].to(dev) for k in STYLE_KEYS})
        assert torch.equal(alone["pooled_output"][0], full["pooled_output"][b])
        assert torch.equal(alone["emotion_outputs"][0], full["emotion_outputs"][b])
    bad = {k: g[k].clone().to(dev) for k in STYLE_KEYS}
    bad["attention_mask"][0, 0] = 0
    with pytest.raises(RuntimeError, match="prefix"):
        m(**bad)
    bad = {k: g[k].clone().to(dev) for k in STYLE_KEYS}
    bad["input_ids"][1, 2] = 10 ** 6
    with pytest.raises(IndexError):
        m(**bad)
    with pytest.raises(RuntimeError):
        m(**{k: g[k] for k in STYLE_KEYS})           # CPU tensors: no CPU path


# ---- training-mode alignment helpers (SURVEY.md s8f rank 4): integer outputs bit-exact vs the reference's numba loops -----

@pytest.mark.parametrize("name", ["align_b3", "align_b2_ties", "align_b4_long"])
def test_alignment_helpers_match_reference_fixture(lib, dev, name):
    from emotivoice_b200 import align
    g = load_golden(name)
    ds, bin_loss, path = align.viterbi_decode(g["log_p_attn"].to(dev), g["text_lengths"].to(dev), g["feats_lengths"].to(dev), return_path=True)
    torch.cuda.synchronize()
    assert torch.equal(path.cpu(), g["paths"])                         # monotonic alignment search: bit-exact (ties included)
    assert torch.equal(ds.cpu(), g["durations"])
    assert abs(float(bin_loss) - float(g["bin_loss"])) <= 1e-6 * abs(float(g["bin_loss"]))
    avg = align.average_by_duration(ds, g["xs"].to(dev), g["text_lengths"].to(dev), g["feats_lengths"].to(dev))
    assert (avg.cpu() - g["averaged"]).abs().max() <= 1e-6
    with pytest.raises(RuntimeError):
        align.viterbi_decode(g["log_p_attn"], g["text_lengths"], g["feats_lengths"])      # CPU tensors: no CPU path


# ==== from here on: tests of code paths that could, in principle, hang (new barrier pipelines, new launch modes); each runs its GPU work
# ==== in a child process under a timeout, and they come last so that everything above has already reported ====================

_KNOB_CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from emotivoice_b200 import synth
from emotivoice_b200.config import default_config
from emotivoice_b200.modules import JETSGenerator
conf = default_config()
m = JETSGenerator(conf).to("cuda:0"); m.load_state_dict(synth.make_state_dict(conf)); m.eval()
z = np.load(sys.argv[2])
keys = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
res = {}
for prec in ("fp32", "tf32", "bf16"):
    m.precision = prec
    for rep in range(3):                      # back-to-back forwards: launches of one forward overlap the tail of the previous one
        out = m(**{k: torch.from_numpy(z[k]).cuda() for k in keys})
    torch.cuda.synchronize()
    res[prec + "_mel"] = out["dec_outputs"].cpu().numpy(); res[prec + "_wav"] = out["wav_predictions"].cpu().numpy()
np.savez(sys.argv[3], **res)
"""


def _check_knobs_bitwise(model, dev, tmp_path, knobs):
    """By default every kernel of the engine is launched with programmatic stream serialization (set-up and weight prefetch of
    launch n+1 overlap the tail of launch n); EV_PDL=0 launches the same kernels without it, their griddepcontrol instructions no-ops.
    EV_VOC_GROUP=0 launches the three parallel ResBlocks of a vocoder stage one convolution at a time, EV_FUSE_RES=0 each ResBlock
    layer as two launches.  None of them reorders any output element's reduction, so every output bit must equal the default mode's;
    a missing griddepcontrol.wait or a tile-shape-dependent result would show up here as a mismatch."""
    import os
    import subprocess
    import sys
    import numpy as np
    from conftest import GOLDEN, ROOT
    src, dst = os.path.join(GOLDEN, "b3_padded.npz"), str(tmp_path / "knobs.npz")
    env = dict(os.environ, **knobs)
    subprocess.run([sys.executable, "-c", _KNOB_CHILD, ROOT, src, dst], env=env, check=True, timeout=240)
    got = np.load(dst)
    g = load_golden("b3_padded")
    try:
        for prec in ("fp32", "tf32", "bf16"):
            model.precision = prec
            out = model(**{k: g[k].to(dev) for k in KEYS})
            assert np.array_equal(out["dec_outputs"].cpu().numpy(), got[prec + "_mel"])
            assert np.array_equal(out["wav_predictions"].cpu().numpy(), got[prec + "_wav"])
    finally:
        model.precision = "fp32"


@pytest.mark.parametrize("knobs", [{"EV_PDL": "0"}, {"EV_VOC_GROUP": "0"}, {"EV_VOC_GROUP": "0", "EV_FUSE_RES": "0"}],
                         ids=["plain_launches", "no_grouped_launches", "no_grouped_no_fused"])
def test_launch_modes_are_bitwise_identical(model, dev, tmp_path, knobs):
    _check_knobs_bitwise(model, dev, tmp_path, knobs)


_ALTERNATE_CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from emotivoice_b200 import synth
from emotivoice_b200.config import default_config
from emotivoice_b200.modules import JETSGenerator
conf = default_config()
m = JETSGenerator(conf).to("cuda:0"); m.load_state_dict(synth.make_state_dict(conf)); m.eval()
batches = [synth.make_batch(lens, seed=11 + i) for i, lens in enumerate(([100], [23, 180, 61, 9], [150, 40], [12], [200, 199, 198, 20, 21, 22, 90, 91]))]
batches = [{k: v.cuda() for k, v in b.items()} for b in batches]
ok = True
for prec in ("fp32", "bf16"):
    m.precision = prec
    first = {}
    for rep in range(6):
        for i, b in enumerate(batches):          # no synchronisation between forwards of different shapes and lengths
            out = m(**b)
            w = out["wav_predictions"]
            if i not in first:
                first[i] = w.clone()
            else:
                ok = ok and bool(torch.equal(w, first[i]))
torch.cuda.synchronize()
print("ALTERNATE_OK" if ok else "ALTERNATE_MISMATCH", flush=True)
"""


def test_back_to_back_batches_of_different_lengths():
    """Programmatic dependent launch lets a kernel start while its predecessors still run; the int32 lengths are written by the first
    kernel of a forward.  A role that read them before griddepcontrol.wait would decode tiles from the PREVIOUS batch's lengths: wrong
    results or -- roles disagreeing on the tile sequence -- a deadlock (that happened once: tensor-core kernel roles that skipped the wait).
    Alternating batches of very different lengths without host synchronisation must reproduce their first results bit for bit."""
    import subprocess
    import sys
    from conftest import ROOT
    r = subprocess.run([sys.executable, "-c", _ALTERNATE_CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ALTERNATE_OK" in r.stdout, (r.stdout[-500:], r.stderr[-1500:])


def test_alignment_module_and_segments_match_reference_fixture(lib, dev):
    """The rest of SURVEY.md s8f rank 4: AlignmentModule.forward (five 3xTF32 convolutions on the tensor cores + the distance /
    log-softmax kernel + the host-built prior) against the unmodified reference module's output (1e-4 on finite entries, the
    -inf pattern identical), and get_random_segments / get_segments bit-exact (same torch RNG calls as the reference)."""
    from emotivoice_b200 import align, synth
    g = load_golden("alignmod_b3")
    mod = align.AlignmentModule(384, 80).to(dev)
    mod.load_state_dict(synth.make_alignment_state_dict(384, 80))
    tl, fl = g["text_lengths"], g["feats_lengths"]
    x_masks = (torch.arange(g["text"].shape[1])[None, :] >= tl[:, None]).to(dev)
    lp = mod(g["text"].to(dev), g["feats"].to(dev), tl, fl, x_masks).cpu()
    ref = g["log_p_attn"]
    fin = torch.isfinite(ref)
    assert torch.equal(fin, torch.isfinite(lp))
    err = (lp[fin] - ref[fin]).abs().max().item()
    print("AlignmentModule max abs err on log_p_attn: %.2e" % err)
    assert err <= 1e-4
    torch.manual_seed(99)
    seg, starts, size = align.get_random_segments(g["z"].to(dev), fl.to(dev), 32)
    assert size == 32 and torch.equal(starts.cpu(), g["starts"]) and torch.equal(seg.cpu(), g["seg"])
    short = align.get_segments(g["z"][:, :, :20].contiguous().to(dev), torch.tensor([0, 3, 19]), 32)
    assert torch.equal(short.cpu(), g["seg_short"])
