"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/joined_*.npz (long text: segments synthesised one by one, their mel
joined and vocoded as one) from the UNMODIFIED reference, and pins oracle/joined_oracle.py against it.

Run in the build container (the GPU box has no reference tree):

    python oracle/make_golden_joined.py

The reference's own ``JETSGenerator`` (jets.py:26) is built with its config.yaml and the seeded state dict of
``emotivoice_b200.synth.make_state_dict``, as in make_golden.py.  Each segment goes through ``ref.am(...)`` as a B=1 call
(what inference_am_vocoder_joint.py:120-129 runs per line); the segments' ``dec_outputs`` are concatenated along time and
``ref.generator(joined.transpose(1, 2))`` vocodes them as one.  The oracle must reproduce every case: durations identical,
mel / wav within 1e-6 relative, as make_golden.py asserts.

Fixtures (ragged per-segment arrays are stored concatenated, with their lengths):
  joined_paragraph.npz  lines 2-5 of the reference's inference text as one paragraph (their inner tokens between one pair of
                        <sos/eos>, 232 tokens), split with split_phonemes(max_phonemes=64) into 5 segments; one speaker, one
                        style / content vector.
  joined_styles.npz     three frontend lines as three segments, each with its own speaker and style / content vector.
Keys: ids, seg_lens, speakers, style, content (S, 768), durations (concatenated per-segment predictions), mel_lens (S,),
joined_mel (sum mel_lens, 80; segment s is rows [sum mel_lens[:s], sum mel_lens[:s+1])), and the joined waveform in windows:
wav_starts (W,) sample offsets and wav_windows (W, 256 * WINDOW_FRAMES), one window at each end of the text and one centred on
every seam, where vocoding the joined mel differs from vocoding the segments one by one.  The whole waveform (256 samples per
frame) would make each fixture over a megabyte; the windows keep it to a few hundred kilobytes.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200.config import default_config          # noqa: E402
from emotivoice_b200 import frontdoor, synth                # noqa: E402
from oracle import joined_oracle                            # noqa: E402
from oracle import refshim                                   # noqa: E402
from oracle.make_golden_prosody import ref_for                # noqa: E402

FRONTDOOR = os.path.join(ROOT, "tests", "golden", "frontdoor")
WINDOW_FRAMES = 24                  # frames of waveform kept around each seam and at each end


def wav_windows(mel_lens, hop=256):
    """Sample offsets of the stored waveform windows: the start, each seam (centred), the end."""
    total, n = int(sum(mel_lens)) * hop, WINDOW_FRAMES * hop
    seams = np.cumsum(mel_lens)[:-1] * hop
    starts = [0] + [min(max(0, int(s) - n // 2), total - n) for s in seams] + [total - n]
    return np.asarray(starts, dtype=np.int64)


def _tables():
    t2i = frontdoor.load_symbol_table(os.path.join(FRONTDOOR, "tokenlist"))
    s2i = frontdoor.load_symbol_table(os.path.join(FRONTDOOR, "speaker2"))
    with open(os.path.join(FRONTDOOR, "inference_text"), encoding="utf-8") as f:
        lines = [frontdoor.parse_line(l) for l in f if l.strip()]
    return t2i, s2i, lines


def _vectors(rng, n):
    return [torch.from_numpy(np.tanh(rng.normal(size=768)).astype(np.float32)) for _ in range(n)]


def cases():
    """name -> (segments as lists of ids, speaker ids, style vectors, content vectors)."""
    t2i, s2i, lines = _tables()
    rng = np.random.default_rng(1250)
    para = [frontdoor.SOS_EOS] + [ph for r in lines[1:5] for ph in r.phonemes[1:-1]] + [frontdoor.SOS_EOS]   # one paragraph
    segs = [[t2i[p] for p in s] for s in frontdoor.split_phonemes(para, max_phonemes=64)]
    st, ct = _vectors(rng, 1)[0], _vectors(rng, 1)[0]
    out = {"paragraph": (segs, [s2i[lines[1].speaker]] * len(segs), [st] * len(segs), [ct] * len(segs))}
    picked = [lines[0], lines[2], lines[3]]
    out["styles"] = ([[t2i[p] for p in r.phonemes] for r in picked], [s2i[r.speaker] for r in picked], _vectors(rng, 3),
                     _vectors(rng, 3))
    return out


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    conf = default_config()
    sd = synth.make_state_dict(conf)
    ref = ref_for(refshim.import_reference_jets(), conf, sd)
    with torch.no_grad():
        for name, (segs, spks, styles, contents) in cases().items():
            ids = [torch.tensor(s, dtype=torch.int64) for s in segs]
            dec = []
            durs = []
            for x, spk, st, ct in zip(ids, spks, styles, contents):
                r = ref.am(x.view(1, -1), torch.tensor([x.numel()]), torch.tensor([spk]), st.view(1, -1).clone(), ct.view(1, -1).clone())
                dec.append(r["dec_outputs"])
                durs.append(r["log_duration_predictions"])
            joined = torch.cat(dec, dim=1)
            wav = ref.generator(joined.transpose(1, 2))
            o = joined_oracle.joined_forward(sd, conf, ids, spks, styles, contents)
            for s, (d, p) in enumerate(zip(durs, o["per_segment"])):
                assert torch.equal(d, p["log_duration_predictions"]), (name, s)
            for k, want, got in (("mel", joined, o["joined_mel"]), ("wav", wav, o["joined_wav"])):
                assert want.shape == got.shape, (name, k, want.shape, got.shape)
                err = (want - got).abs().max().item()
                assert err <= 1e-6 * max(1.0, want.abs().max().item()), (name, k, err)
            starts = wav_windows([d.shape[1] for d in dec])
            np.savez_compressed(
                os.path.join(out_dir, "joined_%s.npz" % name),
                ids=np.concatenate([np.asarray(s, dtype=np.int64) for s in segs]),
                seg_lens=np.asarray([len(s) for s in segs], dtype=np.int64),
                speakers=np.asarray(spks, dtype=np.int64),
                style=torch.stack(styles).numpy(), content=torch.stack(contents).numpy(),
                durations=torch.cat([d[0] for d in durs]).numpy(),
                mel_lens=np.asarray([d.shape[1] for d in dec], dtype=np.int32),
                joined_mel=joined[0].numpy(), wav_starts=starts,
                wav_windows=np.stack([wav[0, 0, s:s + 256 * WINDOW_FRAMES].numpy() for s in starts]))
            print("joined", name, [len(s) for s in segs], "frames %d" % joined.shape[1], "oracle==reference OK")


if __name__ == "__main__":
    main()
