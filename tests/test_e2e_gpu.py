"""End-to-end parity of the CUDA path (through the reference-shaped modules and the C ABI)
against (a) the committed fixtures generated from the unmodified reference and (b) the
oracle, plus size-independent properties at larger sizes.

The default precision mode "fp32" is 3xTF32 on the tensor cores (fp32-accurate); the
plain FFMA path ("fp32_ffma") is held to the same bound.
Tolerances (north_star: "within a stated fp32 mel/waveform tolerance"):
  durations: identical;  mel: max|err| <= 1e-4 * max|mel|;  wav: rms(err) <= 1e-4 * rms(wav).
The fp32 reference's own distance from an fp64 run of the same algorithm is ~1e-6 / 3e-7
(SURVEY.md s4 item 5); the kernels sum in a different order, hence the margin."""
import pytest
import torch

from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import synth, _abi
from oracle import jets_oracle as O

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
MEL_TOL, WAV_TOL = 1e-4, 1e-4


def _run(model, dev, batch):
    out = model(**{k: batch[k].to(dev) for k in KEYS})
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", ["b1_t12", "b1_t50", "b1_t100"])
def test_b1_matches_reference_fixture(model, dev, name):
    g = load_golden(name)
    out = _run(model, dev, g)
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert out["dec_outputs"].shape == g["mel"].shape
    assert out["wav_predictions"].shape == g["wav"].shape
    assert out["wav_predictions"].shape[-1] == 256 * out["dec_outputs"].shape[1]
    assert out["wav_predictions"].dtype == torch.float32 and out["log_duration_predictions"].dtype == torch.int64
    assert rel_max(out["pitch_predictions"].cpu().reshape(1, -1), g["pitch"]) <= MEL_TOL
    assert rel_max(out["energy_predictions"].cpu().reshape(1, -1), g["energy"]) <= MEL_TOL
    e_mel, e_wav = rel_max(out["dec_outputs"].cpu(), g["mel"]), rel_rms(out["wav_predictions"].cpu(), g["wav"])
    print(name, "mel rel-max %.2e wav rms-rel %.2e" % (e_mel, e_wav))
    assert e_mel <= MEL_TOL and e_wav <= WAV_TOL
    assert out["wav_predictions"].abs().max().item() < 1.0
    for k in ("mel_targets", "postnet_outputs", "pitch_targets", "energy_targets", "duration_targets", "output_lengths",
              "log_p_attn", "bin_loss", "z_start_idxs"):
        assert out[k] is None
    assert out["segment_size"] == 32


@pytest.mark.parametrize("name", ["b1_t12", "b1_t100"])
def test_fp32_ffma_mode_matches_reference_fixture(model, dev, name):
    """The plain fp32 FFMA kernels (no tensor cores), precision="fp32_ffma"."""
    g = load_golden(name)
    model.precision = "fp32_ffma"
    try:
        out = _run(model, dev, g)
    finally:
        model.precision = "fp32"
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= MEL_TOL
    assert rel_rms(out["wav_predictions"].cpu(), g["wav"]) <= WAV_TOL


def test_error_vs_fp64_oracle(model, dev, sd, conf):
    """Error against an fp64 run of the algorithm, next to the fp32 reference's own error."""
    g = load_golden("b1_t50")
    out = _run(model, dev, g)
    o64 = O.jets_forward(sd, conf, **{k: g[k] for k in KEYS}, dtype=torch.float64)
    ours = (rel_max(out["dec_outputs"].cpu().double(), o64["dec_outputs"]), rel_rms(out["wav_predictions"].cpu().double(), o64["wav_predictions"]))
    ref32 = (rel_max(g["mel"].double(), o64["dec_outputs"]), rel_rms(g["wav"].double(), o64["wav_predictions"]))
    print("vs fp64: engine mel %.2e wav %.2e | reference-fp32 mel %.2e wav %.2e" % (ours + ref32))
    assert ours[0] <= MEL_TOL and ours[1] <= WAV_TOL


def test_padded_batch_compat_matches_reference_fixture(model, dev):
    """compat_padded_batch=True reproduces the reference's literal padded-batch forward."""
    g = load_golden("b3_padded")
    model.compat_padded_batch = True
    try:
        out = _run(model, dev, g)
    finally:
        model.compat_padded_batch = False
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert out["dec_outputs"].shape == g["mel"].shape
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= MEL_TOL
    assert rel_rms(out["wav_predictions"].cpu(), g["wav"]) <= WAV_TOL


def test_batch_invariant_default_equals_b1_calls(model, dev, sd, conf):
    """Default contract: every item of a padded batch == the reference's B=1 call for it
    (oracle run per utterance) -- and bitwise equal to the engine's own B=1 run."""
    g = load_golden("b3_padded")
    out = _run(model, dev, g)
    per = O.jets_forward_per_utterance(sd, conf, {k: g[k] for k in KEYS})
    for b, r in enumerate(per):
        n = int(g["input_lengths"][b])
        Fb = r["dec_outputs"].shape[1]
        assert torch.equal(out["log_duration_predictions"][b, :n].cpu(), r["log_duration_predictions"][0])
        assert torch.count_nonzero(out["log_duration_predictions"][b, n:]) == 0
        assert int(out["mel_lengths"][b]) == Fb
        assert rel_max(out["dec_outputs"][b, :Fb].cpu(), r["dec_outputs"][0]) <= MEL_TOL
        assert rel_rms(out["wav_predictions"][b, 0, :Fb * 256].cpu(), r["wav_predictions"][0, 0]) <= WAV_TOL
        assert torch.count_nonzero(out["dec_outputs"][b, Fb:]) == 0
        assert torch.count_nonzero(out["wav_predictions"][b, 0, Fb * 256:]) == 0
        single = _run(model, dev, synth.slice_batch(g, b))
        assert torch.equal(single["dec_outputs"][0], out["dec_outputs"][b, :Fb])
        assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256])


def test_generator_forward_matches_reference_fixture(conf, sd, dev, lib):
    """Generator.forward (hifigan/models.py:115-131): (B,80,F) channels-first in, (B,1,256F) out."""
    from emotivoice_b200.modules import Generator
    g = load_golden("voc_b2_f40")
    gen = Generator(conf.model).to(dev)
    gen.load_state_dict({k[len("generator."):]: v for k, v in sd.items() if k.startswith("generator.")})
    wav = gen(g["mel"].to(dev))
    torch.cuda.synchronize()
    assert wav.shape == g["wav"].shape
    assert rel_rms(wav.cpu(), g["wav"]) <= WAV_TOL and rel_max(wav.cpu(), g["wav"]) <= 5e-4
    # legacy (torch < 2.1) checkpoints carry weight_g / weight_v
    legacy = synth.make_state_dict(conf, legacy_weight_norm=True)
    gen.load_state_dict({k[len("generator."):]: v for k, v in legacy.items() if k.startswith("generator.")})
    assert torch.equal(gen(g["mel"].to(dev)), wav)
    gen.remove_weight_norm()
    assert rel_rms(gen(g["mel"].to(dev)).cpu(), g["wav"]) <= WAV_TOL


def test_prompt_tts_forward_alone(conf, sd, dev, lib):
    from emotivoice_b200.modules import PromptTTS
    g = load_golden("b1_t12")
    am = PromptTTS(conf).to(dev)
    am.load_state_dict({k[3:]: v for k, v in sd.items() if k.startswith("am.")})
    out = am(**{k: g[k].to(dev) for k in KEYS})
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    assert rel_max(out["dec_outputs"].cpu(), g["mel"]) <= MEL_TOL


def test_pcm16_matches_numpy_cast(model, dev):
    g = load_golden("b1_t12")
    out = _run(model, dev, g)
    pcm = model.to_pcm16(out["wav_predictions"]).cpu().numpy().reshape(-1)
    assert (pcm == O.to_int16(out["wav_predictions"].cpu())).all()


def test_cfg3_mixed_lengths_batch_properties(model, dev):
    """BASELINE.json configs[2] shape (mixed 20-200 phonemes; 8 items here to bound test
    time): size-independent properties -- per-item bitwise equality with the B=1 run,
    exact x256 lengths, zero padding, |wav| < 1."""
    lens = [200, 20, 57, 133, 96, 164, 31, 75]
    batch = synth.make_batch(lens, seed=4242)
    out = _run(model, dev, batch)
    Fmax = out["dec_outputs"].shape[1]
    assert out["wav_predictions"].shape == (len(lens), 1, 256 * Fmax)
    ml = out["mel_lengths"].cpu().tolist()
    assert max(ml) == Fmax
    assert out["log_duration_predictions"].sum(1).cpu().tolist() == ml
    assert out["wav_predictions"].abs().max().item() < 1.0
    for b in (1, 3, 6):
        single = _run(model, dev, synth.slice_batch(batch, b))
        assert single["dec_outputs"].shape[1] == ml[b]
        assert torch.equal(single["log_duration_predictions"][0], out["log_duration_predictions"][b, :lens[b]])
        assert torch.equal(single["dec_outputs"][0], out["dec_outputs"][b, :ml[b]])
        assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :ml[b] * 256])
        assert torch.count_nonzero(out["wav_predictions"][b, 0, ml[b] * 256:]) == 0


def test_cfg4_vocoder_sweep_point_properties(model, dev):
    """BASELINE.json configs[3]: vocoder-only at (B=4, F=1024): determinism and agreement of
    the batched run with per-item runs (no lengths -> items are independent)."""
    mel = synth.make_mel(4, 1024, seed=9).to(dev)
    w1 = model.generator(mel)
    w2 = model.generator(mel)
    assert w1.shape == (4, 1, 1024 * 256) and torch.equal(w1, w2)
    w_single = model.generator(mel[2:3].contiguous())
    assert torch.equal(w_single[0], w1[2])
    assert torch.isfinite(w1).all() and w1.abs().max().item() < 1.0


def test_engine_reports_its_kernel_launches(model, dev):
    g = load_golden("b1_t12")
    n0 = _abi.launch_count()
    _run(model, dev, g)
    assert _abi.launch_count() - n0 > 100


def test_corpus_runner_is_independent_of_batching(model, dev):
    """SURVEY.md s8e: utterances are independent, so how they are batched / sharded over ranks must not
    change a single PCM sample: synthesize_corpus with batch 1, batch 5 and a 2-rank LPT shard plan."""
    import numpy as np
    from emotivoice_b200 import runner
    rng = np.random.default_rng(5)
    utts = [synth.make_utterance(rng, int(n)) for n in rng.integers(8, 60, size=9)]
    lens = [len(u["ids"]) for u in utts]
    one = runner.synthesize_corpus(model, utts, dev, batch_size=1)
    five = runner.synthesize_corpus(model, utts, dev, batch_size=5)
    shards = runner.plan_shards(lens, 2)
    sharded = {}
    for r in range(2):
        sharded.update(runner.synthesize_corpus(model, utts, dev, batch_size=3, indices=shards[r]))
    assert sorted(one) == sorted(five) == sorted(sharded) == list(range(9))
    for i in range(9):
        assert one[i][1] == five[i][1] == sharded[i][1] and one[i][0].shape == (one[i][1] * 256,)
        assert np.array_equal(one[i][0], five[i][0]) and np.array_equal(one[i][0], sharded[i][0])
        assert one[i][0].dtype == np.int16
        assert one[i][2] == five[i][2] == sharded[i][2] == runner.utterance_digest(one[i][0])
    digest = runner.combine_digests([(i, v[2]) for i, v in one.items()])
    assert digest == runner.combine_digests([(i, v[2]) for i, v in reversed(list(sharded.items()))])


def test_minimal_and_long_sequences(conf, sd, dev, lib):
    """Edge sizes: a 2-phoneme utterance, and an utterance whose frame count exceeds the 5000-row positional
    table the reference starts with (extend_pe, encoder.py:206-237) -- acoustic model only, against the oracle."""
    from emotivoice_b200.modules import PromptTTS
    am = PromptTTS(conf).to(dev)
    am.load_state_dict({k[3:]: v for k, v in sd.items() if k.startswith("am.")})
    tiny = synth.make_batch([2], seed=9)
    out = am(**{k: tiny[k].to(dev) for k in KEYS})
    ref = O.acoustic_model(sd, conf, tiny["inputs_ling"], tiny["input_lengths"], tiny["inputs_speaker"],
                           tiny["inputs_style_embedding"], tiny["inputs_content_embedding"])
    assert torch.equal(out["log_duration_predictions"].cpu(), ref["log_duration_predictions"])
    assert rel_max(out["dec_outputs"].cpu(), ref["dec_outputs"]) <= MEL_TOL
    big = synth.make_batch([900], seed=15)
    out = am(**{k: big[k].to(dev) for k in KEYS})
    ref = O.acoustic_model(sd, conf, big["inputs_ling"], big["input_lengths"], big["inputs_speaker"],
                           big["inputs_style_embedding"], big["inputs_content_embedding"])
    assert out["dec_outputs"].shape[1] > 5000                       # the table had to grow
    assert torch.equal(out["log_duration_predictions"].cpu(), ref["log_duration_predictions"])
    assert rel_max(out["dec_outputs"].cpu(), ref["dec_outputs"]) <= MEL_TOL


def test_bad_inputs_raise_like_the_reference(model, dev):
    """The reference's nn.Embedding raises IndexError for an out-of-range token / speaker id and its mask construction needs
    1 <= length <= T; the engine's kernels index raw memory, so they clamp and report through the status word that the host
    reads with the mel lengths (no extra sync).  Shape errors of the style / content vectors are host checks."""
    good = {k: v.to(dev) for k, v in synth.make_batch([12, 9], seed=4).items()}
    model(**good)
    bad = dict(good, inputs_ling=good["inputs_ling"].clone())
    bad["inputs_ling"][1, 3] = 502
    with pytest.raises(IndexError):
        model(**bad)
    bad = dict(good, inputs_ling=good["inputs_ling"].clone())
    bad["inputs_ling"][0, 0] = -1
    with pytest.raises(IndexError):
        model(**bad)
    with pytest.raises(IndexError):
        model(**dict(good, inputs_speaker=torch.tensor([0, 2014], device=dev)))
    with pytest.raises(RuntimeError):
        model(**dict(good, input_lengths=torch.tensor([12, 0], device=dev)))
    with pytest.raises(RuntimeError):
        model(**dict(good, input_lengths=torch.tensor([13, 9], device=dev)))
    with pytest.raises(RuntimeError):
        model(**dict(good, inputs_style_embedding=good["inputs_style_embedding"][:, :700].contiguous()))
    out = model(**good)          # the engine is still usable afterwards
    assert torch.isfinite(out["wav_predictions"]).all()
