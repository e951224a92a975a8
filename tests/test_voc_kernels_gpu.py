"""The vocoder's granule-planar tensor-core kernels against fp64, at every layer shape and tile plan ev_vocoder issues for the
reference configuration, and the whole vocoder against the fp64 oracle in each of its launch regimes.

Operator level (cases and child process: tests/voc_cases.py; reference and bound: tests/voc_ref.py).  Each kernel family runs
once in its own process under a timeout, so a deadlocked pipeline ends that child and fails its cases, never the suite; no
case is ever run twice.  Every valid output element must satisfy |y - y64| <= tau[mode] * m (+ 2^-9 |y64| for bf16 storage),
m = the sum of the magnitudes of the terms entering it, as well as the bound relative to max|y64| (5e-5 / 3e-3 / 1.2e-2 / 5e-5
for modes 1 / 0 / 2 / 3).  Largest err/m measured on an H100 80GB HBM3 across all operator cases:
    mode 0 (1xTF32)  2^-11.9       tau 2^-9
    mode 1 (3xTF32)  2^-17.9       tau 2^-14
    mode 2 (bf16)    2^-9.2        tau 2^-6
    mode 3 (bf16x3)  2^-17.6       tau 2^-14
Rows past each item's valid length are NaN on input and must be left bit for bit as they were on output.  The bitwise
cross-checks stay where they apply: GP == the time-major TC kernel (modes 0, 1); fused layer == its two launches; grouped
launch == each member's own launch; grouped last layer + gp_sum_div == three accumulating launches.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import voc_cases
import voc_plans
import voc_ref
from conftest import ROOT

pytestmark = pytest.mark.gpu

TIMEOUT = {"conv": 900, "pair": 900, "group": 600, "pair_group": 900, "post": 300}
_ROWS = {}


def _family_rows(family):
    """Runs the family's child once per session; later calls return the same rows (or the same failure)."""
    if family not in _ROWS:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "voc_cases.py"), family], capture_output=True, text=True,
                               timeout=TIMEOUT[family], cwd=ROOT)
            out, tail = r.stdout, "exit %d; stderr: %s" % (r.returncode, r.stderr[-3000:])
        except subprocess.TimeoutExpired as e:
            out = (e.stdout or b"").decode(errors="replace") if isinstance(e.stdout, bytes) else (e.stdout or "")
            tail = "timed out after %d s (a kernel did not finish)" % TIMEOUT[family]
        rows = {}
        for ln in out.splitlines():
            if ln.startswith("{"):
                row = json.loads(ln)
                rows[row["id"]] = row
        _ROWS[family] = (rows, tail)
        print("voc_cases %s: %d rows in %.1f s" % (family, len(rows), time.time() - t0))
    return _ROWS[family]


def _row(family, cid):
    rows, tail = _family_rows(family)
    assert cid in rows, "no result row for %s: %s" % (cid, tail)
    return rows[cid]


def _assert_row(row):
    assert "exception" not in row, row
    if row.get("unsupported"):
        assert row["rc"] != 0, row          # the engine never issues this shape; the kernel must refuse it rather than compute
        return
    assert row["rc"] == 0, row
    assert row["finite"], row
    assert row["pad_untouched"], row
    assert row["bound_ok"], ("err/m %.3g (tau %.3g), rel_max %.3g (bound %.3g)" % (row["err_m"], voc_ref.TAU[row["mode"]], row["rel_max"],
                                                                                   voc_ref.REL_MAX[row["mode"]]), row)
    for k, v in row.items():
        if k.startswith("bitwise"):
            assert v, (k, row)


@pytest.mark.parametrize("cid", voc_cases.case_ids("conv"))
def test_conv1d_gp_against_fp64(cid):
    _assert_row(_row("conv", cid))


@pytest.mark.parametrize("cid", voc_cases.case_ids("pair"))
def test_resblock_gp_against_fp64(cid):
    _assert_row(_row("pair", cid))


@pytest.mark.parametrize("cid", voc_cases.case_ids("group"))
def test_conv1d_gp_group_against_fp64(cid):
    _assert_row(_row("group", cid))


@pytest.mark.parametrize("cid", voc_cases.case_ids("pair_group"))
def test_resblock_gp_group_against_fp64(cid):
    _assert_row(_row("pair_group", cid))


@pytest.mark.parametrize("cid", voc_cases.case_ids("post"))
def test_boundary_kernels(cid):
    row = _row("post", cid)
    assert row["rc"] == 0, row
    if "to_gp" in cid:
        assert row["bitwise_vs_host"], row
        return
    assert row["finite"] and row["pad_zero"], row
    assert row["bound_ok"], ("err/m %.3g > %.3g" % (row["err_m"], voc_cases.TAU_POST), row)


def test_bounds_separate_the_modes():
    """The 1xTF32 results of at least one case fail the fp32-accurate bound: the bounds tell the modes apart.  Prints the
    largest err/m per mode over every operator family."""
    worst = {m: 0.0 for m in voc_cases.MODES}
    for fam in ("conv", "pair", "group", "pair_group"):
        rows, _ = _family_rows(fam)
        for r in rows.values():
            if "err_m" in r and np.isfinite(r["err_m"]):
                worst[r["mode"]] = max(worst[r["mode"]], r["err_m"])
    print("largest err/m per mode:", {m: "%.3g (2^%.1f)" % (v, np.log2(v) if v > 0 else -np.inf) for m, v in worst.items()})
    assert worst[0] > voc_ref.TAU[3]


# ---- the launch list of one ev_vocoder call ------------------------------------------------------------------------------
_KERNEL_MODE = {"tf32": 0, "bf16": 2, "fp32": 3}
POINTS = [  # (B, frames per item): grouped / ungrouped, 64-channel k11 unfused / 128-channel k11 unfused as well
    (1, (1024,)),
    (3, (900, 517, 1)),
    (4, (1050, 613, 255, 2)),
    (8, (700, 1, 150, 37, 260, 9, 64, 129)),
]


@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
def test_launch_list_matches_the_engine(model, lib, dev, prec):
    """tests/voc_plans.engine_launches (the plan-coverage test's list of launches) predicts the number of kernels one
    ev_vocoder call enqueues, in each regime."""
    eng = model._engine()
    try:
        model.precision = prec
        for B, lens in POINTS:
            F = max(lens)
            mel = voc_cases_mel(B, F).to(dev)
            ml = torch.tensor(lens, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            n0 = lib.ev_launch_count()
            eng.vocode(mel, False, ml.data_ptr())
            n1 = lib.ev_launch_count()
            torch.cuda.synchronize()
            assert n1 - n0 == len(voc_plans.engine_launches(lib, B, F, _KERNEL_MODE[prec])), (B, F, prec)
    finally:
        model.precision = "fp32"


def voc_cases_mel(B, F):
    from emotivoice_b200 import synth
    return synth.make_mel(B, F, seed=31 * B + F)


# ---- end to end: the engine's vocoder against the fp64 oracle, per item, per frame --------------------------------------
# per item: the bounds of the vocoder's existing fixture tests; per 256-sample frame: rms error of the frame relative to the
# item's rms (an error confined to an item's end or to one tile cannot hide in the item's rms).  Largest frame error measured on
# an H100 80GB HBM3 over all four points: fp32 3.3e-6, tf32 1.8e-4, bf16 3.5e-3; the frame bounds leave 6-15x of that.
# The fp64 oracle of the 5712 frames took 42 s on 16 CPU threads of the GPU host.
ITEM_RMS = {"fp32": 1e-4, "tf32": 2e-2, "bf16": 2e-2}
ITEM_MAX = {"fp32": 5e-4}
FRAME_RMS = {"fp32": 5e-5, "tf32": 2e-3, "bf16": 2e-2}


@pytest.fixture(scope="module")
def oracle_wavs(sd, conf):
    """fp64 oracle (oracle/jets_oracle.vocoder, hifigan/models.py:115-131) of every item's valid prefix, computed once."""
    from oracle import jets_oracle
    sd64 = jets_oracle._cast_sd(sd, torch.float64)
    t0 = time.time()
    out = {}
    with torch.no_grad():
        for B, lens in POINTS:
            mel = voc_cases_mel(B, max(lens))
            out[B] = [jets_oracle.vocoder(sd64, conf.model, mel[b:b + 1, :, :n].double())[0, 0] for b, n in enumerate(lens)]
    print("fp64 oracle: %d frames in %.1f s on %d CPU threads" % (sum(sum(l) for _, l in POINTS), time.time() - t0, torch.get_num_threads()))
    return out


@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("point", range(len(POINTS)), ids=["B%d_F%d" % (B, max(l)) for B, l in POINTS])
def test_vocoder_against_fp64_oracle(model, dev, oracle_wavs, point, prec):
    B, lens = POINTS[point]
    F = max(lens)
    eng = model._engine()
    try:
        model.precision = prec
        mel = voc_cases_mel(B, F).to(dev)
        ml = torch.tensor(lens, dtype=torch.int32, device=dev)
        wav = eng.vocode(mel, False, ml.data_ptr()).cpu()[:, 0].double()
    finally:
        model.precision = "fp32"
    worst = []
    for b, n in enumerate(lens):
        ref = oracle_wavs[B][b]
        got = wav[b, :n * 256]
        assert bool(torch.isfinite(got).all()), (b, n)
        assert not wav[b, n * 256:].any(), "item %d: waveform not zero past its %d frames" % (b, n)
        rms = ref.pow(2).mean().sqrt().item()
        d = got - ref
        e_rms = d.pow(2).mean().sqrt().item() / rms
        e_max = d.abs().max().item() / ref.abs().max().item()
        e_frame = (d.view(n, 256).pow(2).mean(1).sqrt() / rms).max().item()
        worst.append((b, n, e_rms, e_max, e_frame))
        assert e_rms <= ITEM_RMS[prec] and e_max <= ITEM_MAX.get(prec, 1.0), (prec, b, n, e_rms, e_max)
        assert e_frame <= FRAME_RMS[prec], (prec, b, n, e_frame)
    print("%s B=%d: (item, frames, rel-rms, rel-max, worst frame rms) %s" % (prec, B, ["%d %d %.2e %.2e %.2e" % w for w in worst]))
