"""Pins oracle/align_oracle.py (monotonic alignment search, durations, bin loss, per-token averaging: SURVEY.md s8f rank 4)
against fixtures generated from the reference's own numba functions (alignment.py:90-177) by oracle/make_golden_align.py.
Paths and durations are integers: bit-exact.  The averages restate numba's arithmetic (a sequential float32 sum divided by n in
float64): bit-exact as well.  bin_loss is a float32 mean over frames: 1e-6 relative."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import align_oracle as AO

MAS_FIXTURES = ["mas_t255", "mas_t256", "mas_t257", "mas_t513", "mas_b16", "mas_edges", "mas_ties", "mas_ninf"]
AVG_FIXTURES = ["avg_energy", "avg_logpitch"]


def _np(name):
    return {k: v.numpy() for k, v in load_golden(name).items()}


def mas_inputs(g):
    """The log_p_attn a mas_* fixture was made from, rebuilt bit for bit from its recipe."""
    return AO.band_log_p(g["text_lengths"], g["feats_lengths"], int(g["T_pad"]), int(g["F_pad"]), int(g["seed"]), AO.MAS_KINDS[int(g["kind"])])


def avg_inputs(g):
    """(durations float32, xs float32) of an avg_* fixture: the stored integers times their power-of-two scale, exact."""
    return g["durations"].astype(np.float32), g["xs_q"].astype(np.float32) * np.float32(2.0 ** -int(g["xs_log2_scale"]))


@pytest.mark.parametrize("name", ["align_b3", "align_b2_ties", "align_b4_long"])
def test_alignment_oracle_matches_reference_fixture(name):
    g = _np(name)
    tt, tf = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    ds, bl = AO.viterbi_decode(g["log_p_attn"], tt, tf)
    assert np.array_equal(ds, g["durations"])
    assert abs(float(bl) - float(g["bin_loss"])) <= 1e-6 * abs(float(g["bin_loss"]))
    for b in range(len(tt)):
        path = AO.monotonic_alignment_search(g["log_p_attn"][b, :tf[b], :tt[b]])
        assert np.array_equal(path, g["paths"][b, :tf[b]])
        assert path[0] == 0 and path[-1] == tt[b] - 1 and (np.diff(path) >= 0).all() and (np.diff(path) <= 1).all()      # monotonic, surjective
        assert ds[b].sum() == tf[b]
    assert np.array_equal(AO.average_by_duration(ds, g["xs"], tt, tf), g["averaged"])


@pytest.mark.parametrize("name", MAS_FIXTURES)
def test_mas_oracle_matches_reference_at_training_shapes(name):
    """Paths, durations and per-item bin losses of the reference's search at T_inp 255-513, F up to 1800, B = 16, F < T_inp,
    F == T_inp, F == 1, T == 1, tie-heavy and -inf-holed inputs."""
    g = _np(name)
    lp = mas_inputs(g)
    tt, tf = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    assert lp.shape == (len(tt), int(g["F_pad"]), int(g["T_pad"]))
    ds, bl = AO.viterbi_decode(lp, tt, tf)
    assert np.array_equal(ds, g["durations"].astype(np.float32))
    assert abs(float(bl) - float(g["bin_loss"])) <= 1e-6 * abs(float(g["bin_loss"])) or float(bl) == float(g["bin_loss"])
    for b in range(len(tt)):
        path = AO.monotonic_alignment_search(lp[b, :tf[b], :tt[b]])
        assert np.array_equal(path, g["paths"][b, :tf[b]]) and (g["paths"][b, tf[b]:] == -1).all()
        assert (np.diff(path) >= 0).all() if tf[b] >= tt[b] else (np.diff(path) == 1).all()
        assert ds[b].sum() == tf[b]
        want = -np.float64(lp[b, np.arange(tf[b]), path].astype(np.float64).mean())
        assert float(g["item_bin_loss"][b]) == want or abs(float(g["item_bin_loss"][b]) - want) <= 1e-6 * abs(want)


def test_mas_fixtures_reach_their_edges():
    """The shapes the fixtures were made for are really in them: the strided token loop, F < T_inp, F == 1, T == 1, and
    inputs where the tie rule and -inf cells decide steps of the path."""
    t257, edges = _np("mas_t257"), _np("mas_edges")
    assert t257["text_lengths"].max() > 256 and _np("mas_t513")["text_lengths"].max() == 513
    tl, fl = edges["text_lengths"].tolist(), edges["feats_lengths"].tolist()
    assert any(f < t for t, f in zip(tl, fl)) and any(f == t for t, f in zip(tl, fl)) and 1 in fl and 1 in tl
    assert _np("mas_b16")["text_lengths"].size == 16 and _np("mas_b16")["feats_lengths"].max() == 1800
    for name, what in (("mas_ties", "tie"), ("mas_ninf", "-inf")):
        g = _np(name)
        lp = mas_inputs(g)
        decided = 0
        for b, (t, f) in enumerate(zip(g["text_lengths"].tolist(), g["feats_lengths"].tolist())):
            path, Q = AO.monotonic_alignment_search(lp[b, :f, :t], return_q=True)
            for j in range(f - 1):
                i_b = path[j + 1]
                if what == "tie" and i_b > 0:                   # equal finite predecessors: the rule picks the smaller token
                    decided += bool(Q[i_b - 1, j] == Q[i_b, j] and np.isfinite(Q[i_b, j]))
                elif what == "-inf" and 0 < i_b <= j:           # a reachable predecessor that the -inf cells have cut off
                    decided += bool(np.isneginf(Q[i_b - 1, j]) != np.isneginf(Q[i_b, j]))
            if what == "-inf":
                assert np.isneginf(lp[b, :f, :t]).any()
        assert decided >= 10, (name, decided)


def test_mas_row0_fixture_is_decided_by_the_float32_row_sum():
    """The crafted case: the reference's path, and a float64 row 0 gives a different one (the fixture has teeth)."""
    g = _np("mas_row0")
    lp = g["log_p_attn"][0]
    path = AO.monotonic_alignment_search(lp)
    assert np.array_equal(path, g["paths"][0])
    assert not np.array_equal(g["float64_row0_path"][0], g["paths"][0])
    assert int(np.argmax(path)) == int(np.argmax(g["float64_row0_path"][0])) - 1


@pytest.mark.parametrize("name", AVG_FIXTURES)
def test_average_oracle_equals_reference_bit_for_bit(name):
    """Energy- and log-pitch-like tracks with full float32 mantissas, tokens of 0-600 frames, duration sums below and above
    the feats length, negative durations, lengths past the padded sizes: the oracle equals the reference's numba output exactly,
    and the stored deviation of the reference from the float64 mean is what it says."""
    g = _np(name)
    d, xs = avg_inputs(g)
    tt, tf = g["text_lengths"].tolist(), g["feats_lengths"].tolist()
    assert np.array_equal(AO.average_by_duration(d, xs, tt, tf), g["averaged"])
    m64 = AO.average_by_duration64(d, xs, tt, tf)
    assert np.array_equal(g["averaged_dev"], np.abs(g["averaged"].astype(np.float64) - m64))
    assert (d < 0).any() and (name != "avg_energy" or (any(t > d.shape[1] for t in tt) and any(f > xs.shape[1] for f in tf)))
    assert (g["averaged_dev"] > 0).sum() > 20            # the reference's float32 running sums do round at these magnitudes


def test_alignment_module_oracle_matches_reference_fixture():
    """AlignmentModule.forward (alignment.py:33-56) restated in oracle/align_oracle.py vs the unmodified reference module's
    output (oracle/make_golden_align.py), with the product's host-side beta-binomial prior (the same scipy call as the
    reference's); get_segments vs the reference's segments incl. the t < segment_size zero padding."""
    import torch
    from emotivoice_b200 import synth
    from emotivoice_b200.align import AlignmentModule
    g = load_golden("alignmod_b3")
    sd = synth.make_alignment_state_dict(384, 80)
    tl, fl = g["text_lengths"], g["feats_lengths"]
    T = g["text"].shape[1]
    x_masks = torch.arange(T)[None, :] >= tl[:, None]
    prior = AlignmentModule(384, 80)._generate_prior
    lp = AO.alignment_module_forward(sd, g["text"], g["feats"], tl, fl, x_masks, prior_fn=prior)
    fin = torch.isfinite(g["log_p_attn"])
    assert torch.equal(fin, torch.isfinite(lp)) and (lp[fin] - g["log_p_attn"][fin]).abs().max() <= 1e-5
    assert np.array_equal(AO.get_segments(g["z"].numpy(), g["starts"].numpy(), 32), g["seg"].numpy())
    assert np.array_equal(AO.get_segments(g["z"].numpy()[:, :, :20], np.array([0, 3, 19]), 32), g["seg_short"].numpy())


def test_align_logp64_is_the_module_stage():
    """align_logp64 against the module restatement's distance / log-softmax stage on random float64 inputs (no convolutions)."""
    import torch
    g = torch.Generator().manual_seed(5)
    t, f = torch.randn(2, 7, 16, generator=g, dtype=torch.float64), torch.randn(2, 11, 16, generator=g, dtype=torch.float64)
    tl = torch.tensor([7, 4])
    lp, s_abs, l_abs = AO.align_logp64(t, f, tl)
    score = -torch.norm(f.unsqueeze(2) - t.unsqueeze(1), p=2, dim=3)
    score = score.masked_fill((torch.arange(7)[None, :] >= tl[:, None]).unsqueeze(-2), -np.inf)
    want = torch.log_softmax(score, dim=-1)
    assert torch.equal(torch.isfinite(lp), torch.isfinite(want)) and (lp - want)[torch.isfinite(want)].abs().max() <= 1e-12
    assert s_abs.shape == (2, 11, 7) and l_abs.shape == (2, 11, 1)
