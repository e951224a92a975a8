"""TEST INFRASTRUCTURE ONLY -- the parity oracle of long-text synthesis (``JETSGenerator.forward(join=...)``).

The acoustic model runs on each segment as the reference's B=1 call (jets_oracle.acoustic_model); the segments' mel rows are
concatenated in order, and the vocoder runs once over the joined mel, so HiFi-GAN's receptive field spans every seam
(hifigan/models.py:115-131 on a (1, n_mels, sum F) input).  Pinned against the unmodified reference by
oracle/make_golden_joined.py.
"""
import torch

from oracle import jets_oracle as O


@torch.no_grad()
def joined_forward(sd, conf, segments, speakers, styles, contents, dtype=torch.float32):
    """segments: list of 1-D int64 id tensors; speakers: ints; styles / contents: (768,) tensors, one per segment.
    -> dict(per_segment=[acoustic_model outputs of each B=1 call], joined_mel (1, sum F, n_mels), joined_wav (1, 1, 256 sum F))."""
    sd = O._cast_sd(sd, dtype)
    per = []
    for ids, spk, st, ct in zip(segments, speakers, styles, contents):
        per.append(O.acoustic_model(sd, conf, ids.view(1, -1), torch.tensor([ids.numel()]), torch.tensor([int(spk)]),
                                    st.view(1, -1).to(dtype), ct.view(1, -1).to(dtype)))
    joined = torch.cat([p["dec_outputs"][0] for p in per], dim=0).unsqueeze(0)
    return dict(per_segment=per, joined_mel=joined, joined_wav=O.vocoder(sd, conf.model, joined.transpose(1, 2)))
