"""Host-only checks of the recording-analysis kernel tests (no GPU):

* the representative cases of tests/test_analysis_kernels_gpu.py cover every STFT, pitch and WORLD class of what the analysis
  API accepts (tests/analysis_plans.py), and a list without one of them is reported by the class it leaves uncovered;
* the host helpers agree with the oracles at every representative: ``feats.pitch_frames`` with ``pitch_oracle.frame_count``,
  ``feats.pitch_min_samples`` with the low-cut length and ``feats.world_fft_size`` with ``world_oracle.fft_size``;
* the empty and single-bin bands of the band tables occur where the plans say they do.
"""
import numpy as np
import pytest

import analysis_plans as P
from emotivoice_b200 import feats
from oracle import pitch_oracle as PO
from oracle import world_oracle as W

STFT = [case for case, _ in P.STFT_CASES]


def test_stft_cases_cover_every_class():
    assert P.uncovered(P.stft_classes(), P.stft_covered(STFT)) == []
    for variant, sr, n_mels, fmin, fmax, hop in STFT:
        assert 1 <= hop <= feats.N_FFT and (n_mels is None or 1 <= n_mels <= 128)
    assert sorted({c[5] for c in STFT}) == [1, 2, 255, 256, 257, 300, 511, 1023, 1024]
    assert sorted({c[2] for c in STFT if c[2]}) == [1, 32, 33, 80, 128]
    assert sorted({c[1] for c in STFT}) == list(P.STFT_RATES)


@pytest.mark.parametrize("drop,expect", [
    (("mt", 48000, 128, 0.0, 8000.0, 1024), "most shared memory"),
    (("mt", 8000, 80, 0.0, 8000.0, 1), "hop: lowest (1)"),
    (("taco", 24000, 33, 0.0, None, 1023), "bands: one past a full round (33)"),
    (("mt", 16000, 32, 80.0, 7600.0, 511), "band table with fmin > 0"),
])
def test_an_stft_list_without_a_needed_case_names_the_class_it_leaves(drop, expect):
    left = P.uncovered(P.stft_classes(), P.stft_covered([c for c in STFT if c != drop]))
    assert expect in left, left


def test_the_stft_extremes_are_the_ones_named():
    assert P.stft_smem(1024, 128) == 213248 <= P.SMEM_MAX
    assert max(P.stft_smem(h, m) for h in P.STFT_HOPS for m in P.STFT_MELS) == P.stft_smem(1024, 128)
    assert (P.mt_pad(1), P.mt_pad(255), P.mt_pad(511), P.mt_pad(1023), P.mt_pad(1024)) == (511, 384, 256, 0, 0)


@pytest.mark.parametrize("table,empty,single", [
    ((8000, 80, 0.0, 8000.0), 17, 0),
    ((48000, 128, 0.0, 8000.0), 1, 55),
    ((44100, 128, 0.0, 8000.0), 0, 51),
    ((16000, 80, 0.0, 8000.0), 0, 0),
])
def test_empty_and_single_bin_bands_occur_where_the_plans_say(table, empty, single):
    assert P.band_kinds(*table) == (empty, single)
    bt, bw = feats.band_table(feats.mel_filterbank(table[0], feats.N_FFT, table[1], table[2], table[3]))
    assert int(bt[:, 1].sum()) == bw.size or (bt[:, 1].sum() == 0 and bw.size == 1)
    assert (bt[bt[:, 1] == 0, 0] == 0).all()


def test_every_stft_case_table_is_what_its_reason_says():
    for (variant, sr, n_mels, fmin, fmax, hop), why in P.STFT_CASES:
        if n_mels is None:
            continue
        empty, single = P.band_kinds(sr, n_mels, fmin, fmax)
        if "empty" in why:
            assert empty > 0, why
        if "single-bin" in why:
            assert single > 0, why


def test_pitch_cases_cover_every_class():
    assert P.uncovered(P.pitch_classes(), P.pitch_fields()) == []
    assert sorted(P.PITCH_RATE_CASES) == [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000]
    for fs, hop in P.pitch_configs():
        feats._check_pitch_config(fs, hop)


@pytest.mark.parametrize("drop,expect", [
    (11025, "rate: fs / 50 on MATLAB round's half"),
    (8000, "rate: StoneMask's fs / 12 gate below DIO's ceiling (fs < 9600)"),
])
def test_a_pitch_list_without_a_needed_rate_names_the_class_it_leaves(drop, expect):
    f = P.pitch_fields()
    f["fs"] = f["fs"] - {drop}
    f["config"] = {c for c in f["config"] if c[0] != drop}
    assert expect in P.uncovered(P.pitch_classes(), f)


def test_a_pitch_list_without_the_frame_count_lengths_names_that_class():
    f = P.pitch_fields()
    f["length"] = set()
    assert P.uncovered(P.pitch_classes(), f) == ["length: pyworld's frame count is not n // hop + 1"]


def test_the_pitch_extremes_are_the_ones_named():
    assert P.fix_width(48000, 16) == 85 and P.fix_width(8000, 4096) == 1 and P.fix_width(48000, 4096) == 1
    assert max(P.fix_width(48000, 16), P.fix_width(8000, 16)) == max(P.fix_width(fs, 16) for fs in (8000, 24000, 48000))
    assert (P.lowcut_half(8000), P.lowcut_half(48000)) == (160, 960)
    assert (max(P.band_halves(8000)), max(P.band_halves(48000))) == (159, 956)
    assert 11025 / 50.0 == 220.5 and P.lowcut_half(11025) == 221 != int(11025 / 50.0)
    assert 8000 / 12.0 < 800.0 <= 9600 / 12.0


@pytest.mark.parametrize("fs,hop", P.pitch_configs())
def test_host_pitch_helpers_agree_with_the_oracle(fs, hop):
    fp = feats.pitch_frame_period(fs, hop)
    assert feats.pitch_min_samples(fs) == 2 * PO.lowcut_taps(fs)[0] + 1 == 2 * P.lowcut_half(fs) + 1
    assert len(PO.lowcut_taps(fs)[1]) == feats.pitch_min_samples(fs)
    assert PO.band_half_lengths(fs) == P.band_halves(fs)
    assert P.fix_width(fs, hop) == PO.voice_range_minimum(fp)
    m = feats.pitch_min_samples(fs)
    for n in list(range(m, m + 300)) + [fs, 3 * fs + 7] + FRAME_LENGTHS.get((fs, hop), []):
        assert feats.pitch_frames(n, fs, hop) == PO.frame_count(n, fs, fp) == W.frame_count(n, fs, fp), n


FRAME_LENGTHS = {k: [n + d for n in v for d in (-1, 0, 1)] for k, v in P.FRAME_COUNT_LENGTHS.items()}


def test_the_frame_count_lengths_are_where_pyworld_differs():
    for (fs, hop), ns in P.FRAME_COUNT_LENGTHS.items():
        for n in ns:
            assert feats.pitch_frames(n, fs, hop) == n // hop, n           # one frame fewer than n // hop + 1
            assert feats.pitch_frames(n + 1, fs, hop) == (n + 1) // hop + 1, n
    assert feats.pitch_frames(3328, 22050, 256) == 13


def test_world_cases_cover_every_class():
    assert P.uncovered(P.world_classes(), P.world_fields()) == []
    for rows in P.WORLD_ROW_CASES:
        feats._check_sp2mc(rows - 1, 0.42)
    for a in P.WORLD_ALPHAS:
        feats._check_sp2mc(24, a)
    f = P.world_fields()
    f["rows"] = f["rows"] - {33, 256}
    assert "rows: a fifth round or later" in P.uncovered(P.world_classes(), f)


@pytest.mark.parametrize("fs", sorted({fs for fs, _ in P.pitch_configs()} | set(P.STFT_RATES)))
def test_world_fft_size_is_the_oracles(fs):
    n = feats.world_fft_size(fs)
    assert n == W.fft_size(fs) and n // 2 + 1 in P.WORLD_BIN_CASES


def test_lower_orders_of_the_mel_cepstrum_oracle_are_prefixes_of_higher_ones():
    """freqt's c_0..c_q do not depend on the order past q: the kernel tests slice one order-255 oracle run per frame."""
    sp = np.exp(np.random.default_rng(1).normal(size=513))
    assert np.array_equal(W.sp2mc(sp, 255, 0.42)[:25], W.sp2mc(sp, 24, 0.42))
    assert np.array_equal(W.sp2mc(sp[:3], 255, -0.99)[:1], W.sp2mc(sp[:3], 0, -0.99))


def test_world_hop_edges_are_accepted_frame_periods():
    for fs, hop in P.WORLD_HOP_EDGES:
        feats._check_pitch_config(fs, hop)
        assert 0.25 <= feats.pitch_frame_period(fs, hop) <= 1000.0           # what ev_world_envelope accepts
    assert np.isclose(feats.pitch_frame_period(48000, 16), 1 / 3)
