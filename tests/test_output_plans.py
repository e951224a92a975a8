"""Host-only checks of the output-chain kernel tests (no GPU):

* the representative rates of tests/test_output_kernels_gpu.py cover every resampler, limiter-bank, FLAC rate-code and
  watermark class of the rates ``audio.plan`` accepts, and every extreme (tests/output_plans.py), and a list without one of
  them is reported by the class it leaves uncovered;
* the host's detector bank and hold are the limiter oracle's at every representative rate;
* two facts the loudness kernel's oracle rests on: the K-weighting at 48 kHz is BS.1770-4's coefficient table, and a
  full-scale 1 kHz sine reads -3.01 LUFS (the standard's own calibration) at 8, 16 and 48 kHz.
"""
import numpy as np
import pytest

import output_plans as P
from emotivoice_b200 import audio
from oracle import limiter_oracle, loudness_oracle


def test_every_accepted_rate_is_enumerated():
    p = P.plans()
    codes = [q["flac"] for q in p.values()]
    assert len(p) == 6929 and min(p) == 4000 and max(p) == 192000
    assert (codes.count(12), codes.count(13), codes.count(14), codes.count(0)) == (182, 4400, 1675, 661)
    assert sum(q["flac_kind"] == "standard" for q in p.values()) == len(audio.FLAC_STANDARD_RATES)
    assert all(max(q["up"], q["down"]) <= audio.MAX_FACTOR for q in p.values())
    for rate in (4001, 16001, 191999):               # ratios whose factors exceed 1024
        with pytest.raises(ValueError):
            audio.plan(rate, "pcm16", P.SOURCE_RATE)


def test_representative_rates_cover_every_class():
    assert P.uncovered(P.REPRESENTATIVE_RATES) == []
    p = P.plans()
    assert set(P.REPRESENTATIVE_RATES) <= set(p)
    want = {4000: (1, 4), 4016: (251, 1000), 8000: (1, 2), 11025: (441, 640), 12000: (3, 4), 15625: (125, 128), 16000: (1, 1),
            16368: (1023, 1000), 65600: (41, 10), 127625: (1021, 128), 131072: (1024, 125), 192000: (12, 1)}
    assert {r: (p[r]["up"], p[r]["down"]) for r in P.REPRESENTATIVE_RATES} == want


def test_the_extremes_are_the_ones_named():
    p = P.plans()
    assert (p[4000]["taps"], p[4000]["window"]) == (81, 1101)
    assert (p[4016]["taps"], p[4016]["window"]) == (80, 1096)
    assert p[16368]["smem"] == 87016 and max(q["smem"] for q in p.values()) == 87016
    assert p[131072]["smem"] < 160 * 1024                 # what launch_audio_out lets audio_out_kernel use
    assert (p[4000]["bank"], p[4000]["hold"]) == ((12, 101), 50) and p[4016]["bank"] == (12, 101)
    assert (p[15625]["bank"], p[15625]["hold"]) == ((12, 43), 21)
    assert {q["bank"] for q in p.values() if q["bank"][0] == 11} == {(11, 21)}
    assert [p[r]["flac"] for r in (4000, 4016, 12000, 65600, 127625, 131072, 192000)] == [12, 13, 12, 14, 0, 0, 3]


@pytest.mark.parametrize("drop", [65600, 131072, 4000, 16368, 15625, 16000])
def test_a_list_without_a_needed_rate_names_the_class_it_leaves(drop):
    left = P.uncovered(set(P.REPRESENTATIVE_RATES) - {drop})
    assert left, drop
    expect = {65600: "FLAC rate code 14", 131072: "largest up", 4000: "lowest rate", 16368: "most shared memory",
              15625: "narrowest low-passed limiter bank", 16000: "resampler copy"}[drop]
    assert expect in left, left


@pytest.mark.parametrize("rate", sorted(P.REPRESENTATIVE_RATES))
def test_host_bank_is_the_oracles_filter_at_every_representative_rate(rate):
    bank, hold = audio.limit_bank(P.SOURCE_RATE, rate)
    h, c, phases = limiter_oracle.detector_filter(P.SOURCE_RATE, rate)
    R = limiter_oracle.oversampling(P.SOURCE_RATE)
    assert hold == limiter_oracle.hold(P.SOURCE_RATE, rate) and bank.shape == (len(phases), 2 * c + 1)
    for row, ph in zip(bank, phases):
        want = h[ph::R]
        assert np.array_equal(row[:len(want)], want.astype(np.float32)) and not row[len(want):].any()


def test_k_weighting_at_48k_is_the_standards_table():
    k = audio.k_weighting(48000)
    t = loudness_oracle.TABLE_48K
    table = np.array(list(t["shelf_b"]) + list(t["shelf_a"][1:]) + list(t["hp_b"]) + list(t["hp_a"][1:]))
    assert np.max(np.abs(k - table)) <= 1e-12


@pytest.mark.parametrize("sr", [8000, 16000, 48000])
def test_full_scale_1khz_sine_reads_minus_3_01_lufs(sr):
    x = np.sin(2 * np.pi * 1000.0 * np.arange(5 * sr) / sr)
    assert abs(loudness_oracle.integrated_loudness(x, sr) + 3.01) <= 0.1
