"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/prosody_*.npz (speaking-rate, pitch and energy
controls) from the UNMODIFIED reference, and pins oracle/prosody_oracle.py against it.

Run in the build container (the GPU box has no reference tree):

    python oracle/make_golden_prosody.py

The reference's own ``JETSGenerator`` (jets.py:26) is built with its config.yaml and the seeded state dict
of ``emotivoice_b200.synth.make_state_dict``.  Its inference branch (model_open_source.py:102-163) is then
driven through the reference's own submodule objects, with the controls inserted where they act:
``length_regulator(..., alpha=a)`` (alignment.py:180-183, the rate control the inference branch does not
pass on) and ``p * p_scale + p_shift`` / ``e * e_scale + e_shift`` on the predictions just before
``pitch_embed`` / ``energy_embed`` (:131-134).  With neutral controls that driver must equal
``generator(**kw)`` bit for bit; the oracle must reproduce every case (durations and frame counts
identical, mel / wav within 1e-6 relative, as make_golden.py asserts).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200.config import default_config          # noqa: E402
from emotivoice_b200 import synth                           # noqa: E402
from oracle import prosody_oracle as O                        # noqa: E402
from oracle import refshim                                   # noqa: E402

KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
CONTROLS = ("duration_scale", "pitch_shift", "energy_scale")
NEUTRAL = dict(duration_scale=1.0, pitch_shift=0.0, energy_scale=1.0)

# name: (phoneme counts, input seed, per-item controls {kwarg: list}, literal padded batch?, duration-head bias)
CASES = {
    "a050": ([100], synth.SEED, dict(duration_scale=[0.5]), False, None),         # exact products
    "a080": ([100], synth.SEED, dict(duration_scale=[0.8]), False, None),
    "a125": ([100], synth.SEED, dict(duration_scale=[1.25]), False, None),
    "a200": ([50], 1242, dict(duration_scale=[2.0]), False, None),               # the 50-phoneme input keeps the file small
    "p_up4": ([50], 1242, dict(pitch_shift=[4.0]), False, None),
    "p_down4": ([50], 1242, dict(pitch_shift=[-4.0]), False, None),
    "e070": ([50], 1242, dict(energy_scale=[0.7]), False, None),
    "e130": ([50], 1242, dict(energy_scale=[1.3]), False, None),
    "combined": ([50], 1242, dict(duration_scale=[0.8], pitch_shift=[-4.0], energy_scale=[1.3]), False, None),
    # three items, each its own B=1 reference call (the engine's default batch contract); item 1 neutral
    "mixed3": ([9, 23, 14], 1243, dict(duration_scale=[0.8, 1.0, 1.25], pitch_shift=[4.0, 0.0, -4.0],
                                       energy_scale=[1.0, 1.0, 0.7]), False, None),
    # a duration head biased to predict zero everywhere: the all-zero guard writes 1, not alpha (alignment.py:187-191)
    "zero_dur": ([12], 1240, dict(duration_scale=[0.75]), False, -30.0),
    # the reference's literal padded forward with ds * alpha[:, None] and per-item affine
    "padded": ([9, 23, 14], 1243, dict(duration_scale=[0.8, 1.25, 0.5], pitch_shift=[2.0, 0.0, -3.0],
                                       energy_scale=[1.1, 1.0, 0.9]), True, None),
}
ZERO_FRAMES = ("zero_frames", [12], 1240, dict(duration_scale=[0.01]))   # scaled to 0 frames: the reference raises


def drive_reference(gen, batch, table):
    """The reference's inference branch through its own submodules, controls inserted.  table: (B,5) or None."""
    am = gen.am
    ling, lens, spk = batch["inputs_ling"], batch["input_lengths"], batch["inputs_speaker"]
    style, content = batch["inputs_style_embedding"], batch["inputs_content_embedding"]
    B, T = ling.shape
    src_mask = am.get_mask_from_lengths(lens)
    x, _ = am.encoder(am.src_word_emb(ling), ~src_mask.unsqueeze(-2))
    s = am.spk_tokenizer(spk)
    x = torch.concat([x, s.unsqueeze(1).expand(B, T, -1), style.unsqueeze(1).expand(B, T, -1),
                      content.unsqueeze(1).expand(B, T, -1)], dim=-1)
    x = am.embed_projection1(x)
    p_outs = am.pitch_predictor(x, src_mask.unsqueeze(-1))
    e_outs = am.energy_predictor(x, src_mask.unsqueeze(-1))
    d_outs = am.duration_predictor.inference(x, src_mask.unsqueeze(-1))
    p_in, e_in, alpha = p_outs, e_outs, 1.0
    if table is not None:
        p_in = p_outs * table[:, 1:2] + table[:, 2:3]
        e_in = e_outs * table[:, 3:4] + table[:, 4:5]
        alpha = float(table[0, 0]) if B == 1 else table[:, 0:1]
    x = x + am.pitch_embed(p_in.unsqueeze(1)).transpose(1, 2) + am.energy_embed(e_in.unsqueeze(1)).transpose(1, 2)
    x = am.length_regulator(x, d_outs, None, ~src_mask, alpha=alpha)
    x, _ = am.decoder(x, None)
    mel = am.to_mel(x)
    return dict(dec_outputs=mel, log_duration_predictions=d_outs, pitch_predictions=p_outs.squeeze(), energy_predictions=e_outs.squeeze(),
                wav_predictions=gen.generator(mel.transpose(1, 2)))


def assert_out_of_band(d, alpha):
    """The engine counts trunc(fl32(exact sum of fl32(d * alpha))); the reference's fp32 cascade sum agrees unless the exact
    sum lies within a few fp32 ulps of an integer.  No fixture item may sit in that band, except where every product is
    exact (alpha a power of two, or the all-zero guard's ones)."""
    ds = d.float() * torch.tensor(alpha, dtype=torch.float32).reshape(-1, 1)
    for row, a in zip(ds, alpha):
        if float(row.sum()) == 0 or float(np.float32(a)) == 2.0 ** round(np.log2(a)):
            continue
        s = float(row.double().sum())
        ulp, gap = float(np.spacing(np.float32(s))), abs(s - round(s))
        assert gap > 8 * ulp, "sum %r within %.1f ulp of an integer" % (s, gap / ulp)


def ref_for(JETS, conf, sd):
    ref = JETS(refshim.load_reference_config(conf.n_vocab, conf.n_speaker)).eval()
    ref.load_state_dict(sd, strict=True)
    return ref


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    conf = default_config()
    sd = synth.make_state_dict(conf)
    JETS = refshim.import_reference_jets()
    ref = ref_for(JETS, conf, sd)
    with torch.no_grad():
        # the driver is the reference's own forward when the controls are neutral
        batch = synth.make_batch([50], seed=1242)
        want = ref(**{k: v.clone() for k, v in batch.items()})
        got = drive_reference(ref, {k: v.clone() for k, v in batch.items()}, None)
        for k in ("dec_outputs", "wav_predictions", "log_duration_predictions", "pitch_predictions", "energy_predictions"):
            assert torch.equal(want[k], got[k]), k
        print("driver == generator(**kw) with neutral controls OK")

        for name, (lens, seed, controls, literal, dur_bias) in CASES.items():
            B = len(lens)
            batch = synth.make_batch(lens, seed=seed)
            csd = dict(sd)
            if dur_bias is not None:
                csd["am.duration_predictor.linear.bias"] = torch.full_like(sd["am.duration_predictor.linear.bias"], dur_bias)
            r = ref if dur_bias is None else ref_for(JETS, conf, csd)
            full = {c: controls.get(c, [NEUTRAL[c]] * B) for c in CONTROLS}
            arrays = {k: v.numpy() for k, v in batch.items()}
            arrays.update({c: np.asarray(full[c], dtype=np.float64) for c in CONTROLS})
            arrays["literal"] = np.asarray(literal)
            if dur_bias is not None:
                arrays["dur_bias"] = np.asarray(dur_bias, dtype=np.float32)
            if literal:
                table = O.prosody_table(B, **full)
                want = drive_reference(r, {k: v.clone() for k, v in batch.items()}, table)
                o = O.jets_forward(csd, conf, **batch, **full)
                assert torch.equal(want["log_duration_predictions"], o["log_duration_predictions"]), name
                assert int(o["mel_lens"].max()) == want["dec_outputs"].shape[1], name
                assert_out_of_band(o["log_duration_predictions"], full["duration_scale"])
                for k in ("dec_outputs", "wav_predictions"):
                    err = (want[k] - o[k]).abs().max().item()
                    assert err <= 1e-6 * max(1.0, want[k].abs().max().item()), (name, k, err)
                arrays.update(durations=want["log_duration_predictions"].numpy(), mel_lens=o["mel_lens"].numpy(),
                              pitch=want["pitch_predictions"].reshape(B, -1).numpy(),
                              energy=want["energy_predictions"].reshape(B, -1).numpy(),
                              mel=want["dec_outputs"].numpy(), wav=want["wav_predictions"].numpy())
            else:
                per = O.jets_forward_per_utterance(csd, conf, batch, controls=full)
                for b in range(B):
                    one = synth.slice_batch(batch, b)
                    kw = {c: [full[c][b]] for c in CONTROLS}
                    want = drive_reference(r, {k: v.clone() for k, v in one.items()}, O.prosody_table(1, **kw))
                    o = per[b]
                    assert torch.equal(want["log_duration_predictions"], o["log_duration_predictions"]), (name, b)
                    assert int(o["mel_lens"][0]) == want["dec_outputs"].shape[1], (name, b)
                    assert_out_of_band(o["log_duration_predictions"], kw["duration_scale"])
                    for k in ("dec_outputs", "wav_predictions"):
                        err = (want[k] - o[k]).abs().max().item()
                        assert err <= 1e-6 * max(1.0, want[k].abs().max().item()), (name, b, k, err)
                    arrays.update({"durations_%d" % b: want["log_duration_predictions"].numpy(),
                                   "mel_lens_%d" % b: o["mel_lens"].numpy(),
                                   "pitch_%d" % b: want["pitch_predictions"].reshape(1, -1).numpy(),
                                   "energy_%d" % b: want["energy_predictions"].reshape(1, -1).numpy(),
                                   "mel_%d" % b: want["dec_outputs"].numpy(), "wav_%d" % b: want["wav_predictions"].numpy()})
                    if dur_bias is not None:
                        assert int(want["log_duration_predictions"].abs().sum()) == 0, name
            np.savez_compressed(os.path.join(out_dir, "prosody_%s.npz" % name), **arrays)
            print("prosody", name, lens, "oracle==reference OK")

        name, lens, seed, controls = ZERO_FRAMES
        batch = synth.make_batch(lens, seed=seed)
        table = O.prosody_table(1, **controls)
        raised = False
        try:
            drive_reference(ref, {k: v.clone() for k, v in batch.items()}, table)
        except RuntimeError:
            raised = True
        assert raised, "the reference was expected to raise on a zero-frame utterance"
        arrays = {k: v.numpy() for k, v in batch.items()}
        arrays.update(duration_scale=np.asarray(controls["duration_scale"]), pitch_shift=np.zeros(1), energy_scale=np.ones(1),
                      reference_raises=np.asarray(True))
        np.savez_compressed(os.path.join(out_dir, "prosody_%s.npz" % name), **arrays)
        print("prosody", name, "reference raises RuntimeError OK")


if __name__ == "__main__":
    main()
