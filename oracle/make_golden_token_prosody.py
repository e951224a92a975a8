"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/token_prosody_*.npz (phoneme-level prosody controls and
caller-given durations, pitch and energy) from the UNMODIFIED reference, and pins oracle/token_prosody_oracle.py
against it.

Run in the build container (the GPU box has no reference tree):

    python oracle/make_golden_token_prosody.py

The reference's own ``JETSGenerator`` (jets.py:26) is built with its config.yaml and the seeded state dict of
``emotivoice_b200.synth.make_state_dict``.  Its inference branch (model_open_source.py:102-163) is driven through the
reference's own submodule objects, the way its training branch feeds externally computed values (:113-140):
``length_regulator(x, ds, None, ~src_mask, alpha=<(B,T) tensor>)`` with caller durations ``ds`` in place of d_outs
(alignment.py:180-191), and per-token affine tracks p * p_scale + p_shift / e * e_scale + e_shift (on the caller's tracks
where given) into ``pitch_embed`` / ``energy_embed``.  The oracle must reproduce every case: durations and frame counts
identical, mel / wav within 1e-6 relative, as make_golden.py asserts.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200.config import default_config          # noqa: E402
from emotivoice_b200 import synth                           # noqa: E402
from oracle import token_prosody_oracle as O                  # noqa: E402
from oracle import refshim                                   # noqa: E402
from oracle.make_golden_prosody import ref_for                # noqa: E402

KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
CONTROLS = ("duration_scale", "pitch_shift", "energy_scale")
GIVEN = ("durations", "pitch", "energy")


def ramp(lens, T, fn, neutral):
    """(B,T) float64 table: fn(b, t) on each item's valid tokens, neutral on its pads."""
    a = np.full((len(lens), T), neutral, dtype=np.float64)
    for b, n in enumerate(lens):
        for t in range(n):
            a[b, t] = fn(b, t)
    return a


def cases():
    """name -> (phoneme counts, input seed, controls {kwarg: value}, literal padded batch?)."""
    out = {}
    # a lengthened pause (token 40, x3) and a sped-up word (tokens 10..14, duration scale 0.7) in one utterance
    out["pause_word"] = ([100], synth.SEED, dict(duration_scale=ramp([100], 100, lambda b, t: 3.0 if t == 40 else
                                                                    (0.7 if 10 <= t <= 14 else 1.0), 1.0)), False)
    # +5 semitones on tokens 20..27, energy x1.2 on the same span
    out["pitch_span"] = ([50], 1242, dict(pitch_shift=ramp([50], 50, lambda b, t: 5.0 if 20 <= t <= 27 else 0.0, 0.0),
                                          energy_scale=ramp([50], 50, lambda b, t: 1.2 if 20 <= t <= 27 else 1.0, 1.0)), False)
    # caller durations: item 0 with zeros in it (some tokens get no frame), item 1 all zero (the guard gives each token 1)
    rng = np.random.default_rng(31)
    d = rng.integers(0, 9, size=(2, 23)).astype(np.int64)
    d[0, [3, 4, 11]] = 0
    d[1] = 0
    d[0, 17:] = 0                                                # item 0 has 17 phonemes; its pads are ignored anyway
    d[0, 18] = 7
    out["caller_dur"] = ([17, 23], 1244, dict(durations=d, duration_scale=[1.3, 0.75]), False)
    # caller pitch / energy tracks (normalised units), with a per-token pitch shift on top
    p = np.sin(np.arange(30) / 3.0)[None, :] * 1.5
    e = np.cos(np.arange(30) / 4.0)[None, :] * 0.8 + 0.2
    out["caller_pe"] = ([30], 1245, dict(pitch=p.astype(np.float32), energy=e.astype(np.float32),
                                         pitch_shift=ramp([30], 30, lambda b, t: -3.0 if t < 6 else 0.0, 0.0)), False)
    # three items, each its own B=1 call: per-token rate, per-item only, per-token pitch + energy
    lens = [9, 23, 14]
    out["mixed3"] = (lens, 1243, dict(
        duration_scale=ramp(lens, 23, lambda b, t: [1.0 + 0.1 * (t % 4), 1.25, 1.0][b] if b != 2 else 1.0, 1.0),
        pitch_shift=ramp(lens, 23, lambda b, t: [0.0, -2.0, 0.5 * t][b], 0.0),
        energy_scale=ramp(lens, 23, lambda b, t: [1.0, 1.0, 0.9 + 0.02 * t][b], 1.0)), False)
    # the reference's literal padded forward with per-token scales and caller durations; garbage in the pads is ignored
    d = rng.integers(1, 7, size=(3, 23)).astype(np.int64)
    for b, n in enumerate(lens):
        d[b, n:] = 99
    out["padded"] = (lens, 1243, dict(durations=d, duration_scale=ramp(lens, 23, lambda b, t: 0.75 + 0.05 * (t % 7), 1.0),
                                      pitch_shift=ramp(lens, 23, lambda b, t: 2.0 if t % 5 == 0 else 0.0, 0.0)), True)
    return out


ZERO_FRAMES = ("zero_frames", [12], 1240, dict(durations=np.array([[1] + [0] * 11], dtype=np.int64), duration_scale=[0.5]))


def drive_reference(gen, batch, table, durations=None, pitch=None, energy=None):
    """The reference's inference branch through its own submodules, with a (B,T,5) table (or None) and caller values
    (pads already neutral / zero)."""
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
    p_in = p_outs if pitch is None else pitch
    e_in = e_outs if energy is None else energy
    ds = d_outs if durations is None else durations
    alpha = 1.0
    if table is not None:
        p_in = p_in * table[..., 1] + table[..., 2]
        e_in = e_in * table[..., 3] + table[..., 4]
        alpha = table[..., 0]
    x = x + am.pitch_embed(p_in.unsqueeze(1)).transpose(1, 2) + am.energy_embed(e_in.unsqueeze(1)).transpose(1, 2)
    x = am.length_regulator(x, ds.clone(), None, ~src_mask, alpha=alpha)
    x, _ = am.decoder(x, None)
    mel = am.to_mel(x)
    return dict(dec_outputs=mel, log_duration_predictions=d_outs, pitch_predictions=p_outs.squeeze(), energy_predictions=e_outs.squeeze(),
                wav_predictions=gen.generator(mel.transpose(1, 2)))


def assert_out_of_band(ds_int, alpha):
    """The engine counts trunc(fl32(exact sum of fl32(d * alpha))); the reference's fp32 cascade sum agrees unless the exact
    sum lies within a few fp32 ulps of an integer.  No fixture item may sit in that band, except where every product is
    exact.  ds_int (B,T) int64 (zero pads); alpha None or (B,T) float32."""
    a = torch.ones(ds_int.shape) if alpha is None else alpha
    ds = ds_int.float() * a
    for row, d, ar in zip(ds, ds_int, a):
        if float(row.sum()) == 0 or torch.equal(row.double(), d.double() * ar.double()):
            continue
        s = float(row.double().sum())
        ulp, gap = float(np.spacing(np.float32(s))), abs(s - round(s))
        assert gap > 8 * ulp, "sum %r within %.1f ulp of an integer" % (s, gap / ulp)


def _tensors(lens, T, controls):
    table = O.token_table(lens, T, *(controls.get(c) for c in CONTROLS))
    pad = torch.arange(T).unsqueeze(0) >= torch.tensor(lens).unsqueeze(1)
    given = {k: torch.as_tensor(controls[k]).masked_fill(pad, 0) for k in GIVEN if k in controls}
    return table, given


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    conf = default_config()
    sd = synth.make_state_dict(conf)
    JETS = refshim.import_reference_jets()
    ref = ref_for(JETS, conf, sd)
    with torch.no_grad():
        for name, (lens, seed, controls, literal) in cases().items():
            B, T = len(lens), max(lens)
            batch = synth.make_batch(lens, seed=seed)
            arrays = {k: v.numpy() for k, v in batch.items()}
            for k, v in controls.items():
                arrays[k] = np.asarray(v)
            arrays["literal"] = np.asarray(literal)
            if literal:
                table, given = _tensors(lens, T, controls)
                want = drive_reference(ref, {k: v.clone() for k, v in batch.items()}, table, **given)
                o = O.jets_forward(sd, conf, **batch, **controls)
                assert torch.equal(want["log_duration_predictions"], o["log_duration_predictions"]), name
                assert int(o["mel_lens"].max()) == want["dec_outputs"].shape[1], name
                assert_out_of_band(given.get("durations", o["log_duration_predictions"]), None if table is None else table[..., 0])
                for k in ("dec_outputs", "wav_predictions"):
                    err = (want[k] - o[k]).abs().max().item()
                    assert err <= 1e-6 * max(1.0, want[k].abs().max().item()), (name, k, err)
                arrays.update(pred_durations=want["log_duration_predictions"].numpy(), mel_lens=o["mel_lens"].numpy(),
                              pred_pitch=want["pitch_predictions"].reshape(B, -1).numpy(),
                              mel=want["dec_outputs"].numpy(), wav=want["wav_predictions"].numpy())
            else:
                per = O.jets_forward_per_utterance(sd, conf, batch, controls=controls)
                for b in range(B):
                    n = lens[b]
                    one = synth.slice_batch(batch, b)
                    kw = O.item_controls(controls, b, n)
                    table, given = _tensors([n], n, kw)
                    want = drive_reference(ref, {k: v.clone() for k, v in one.items()}, table, **given)
                    o = per[b]
                    assert torch.equal(want["log_duration_predictions"], o["log_duration_predictions"]), (name, b)
                    assert int(o["mel_lens"][0]) == want["dec_outputs"].shape[1], (name, b)
                    assert_out_of_band(given.get("durations", o["log_duration_predictions"]), None if table is None else table[..., 0])
                    for k in ("dec_outputs", "wav_predictions"):
                        err = (want[k] - o[k]).abs().max().item()
                        assert err <= 1e-6 * max(1.0, want[k].abs().max().item()), (name, b, k, err)
                    arrays.update({"pred_durations_%d" % b: want["log_duration_predictions"].numpy(),
                                   "mel_lens_%d" % b: o["mel_lens"].numpy(),
                                   "pred_pitch_%d" % b: want["pitch_predictions"].reshape(1, -1).numpy(),
                                   "mel_%d" % b: want["dec_outputs"].numpy(), "wav_%d" % b: want["wav_predictions"].numpy()})
            np.savez_compressed(os.path.join(out_dir, "token_prosody_%s.npz" % name), **arrays)
            print("token prosody", name, lens, "oracle==reference OK")

        name, lens, seed, controls = ZERO_FRAMES
        batch = synth.make_batch(lens, seed=seed)
        table = O.token_table(lens, max(lens), duration_scale=controls["duration_scale"])
        raised = False
        try:
            drive_reference(ref, {k: v.clone() for k, v in batch.items()}, table, durations=torch.as_tensor(controls["durations"]))
        except RuntimeError:
            raised = True
        assert raised, "the reference was expected to raise on a zero-frame utterance"
        arrays = {k: v.numpy() for k, v in batch.items()}
        arrays.update({k: np.asarray(v) for k, v in controls.items()})
        arrays["reference_raises"] = np.asarray(True)
        np.savez_compressed(os.path.join(out_dir, "token_prosody_%s.npz" % name), **arrays)
        print("token prosody", name, "reference raises RuntimeError OK")


if __name__ == "__main__":
    main()
