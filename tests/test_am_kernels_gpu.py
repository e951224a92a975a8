"""The acoustic model's tensor-core kernels against fp64, at every layer shape, kernel MODE, K-split factor and tile plan
ev_am_phase1 / ev_am_phase2 issue for the reference configuration, and at item lengths on the tile edges.

Operator level (cases and child process: tests/am_cases.py; reference and bound: tests/am_ref.py; launch list:
tests/am_plans.py).  Each kernel family runs once in its own process under a timeout, so a deadlocked pipeline ends that child
and fails its cases, never the suite; no case is ever run twice.  Every valid output element must satisfy
|y - y64| <= tau[MODE] * m, m = the sum of the magnitudes of the terms entering it (through the softmax for attention), with
tau = 2^-9 (1xTF32), 2^-14 (3xTF32, bf16x3), 2^-6 (bf16), as well as the bound relative to max|y64| each mode has always been
held to.  Rows past each item are NaN on input; conv rows past an item must come out as exact zeros.  Bitwise: two runs; the
in-place residual (wo, ffn2) against the out-of-place one; an item of a ragged batch of 32 against its own batch-1 launch.

Largest err/m measured on an H100 80GB HBM3 (the bounds are derived, not fitted: at S = 16 a 3xTF32 ffn2 slice is a chain of
288 products and the reduce adds 16 slices, <= ~300 * 2^-24 = 2^-15.8 of m in fp32 accumulation even in the worst case):
    conv1d_tc    MODE 0 (1xTF32) 2^-13.1   MODE 1 (3xTF32) 2^-21.1   MODE 2 (bf16) 2^-10.0   MODE 3 (bf16x3) 2^-19.0
    attention_tc MODE 0 (1xTF32) 2^-11.0   MODE 1 (3xTF32) 2^-19.8
The two child processes took 13 s (65 conv cases) and 16 s (20 attention cases) including their fp64 references on the GPU
host's 16 CPU threads; the whole file about 35 s.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import am_cases
import am_plans
import voc_ref
from conftest import ROOT

pytestmark = pytest.mark.gpu

TIMEOUT = {"tc": 1200, "attn": 600, "style": 1200}
_ROWS = {}


def _family_rows(family):
    """Runs the family's child once per session; later calls return the same rows (or the same failure)."""
    if family not in _ROWS:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "am_cases.py"), family], capture_output=True, text=True,
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
        print("am_cases %s: %d rows in %.1f s" % (family, len(rows), time.time() - t0))
    return _ROWS[family]


def _row(family, cid):
    rows, tail = _family_rows(family)
    assert cid in rows, "no result row for %s: %s" % (cid, tail)
    return rows[cid]


def _assert_row(row):
    assert "exception" not in row, row
    assert row["rc"] == 0, row
    assert row["finite"], row
    assert row.get("pad_zero", True), row
    assert row["bound_ok"], ("err/m %.3g (tau %.3g), rel_max %.3g" % (row["err_m"], voc_ref.TAU[row["mode"]], row["rel_max"]), row)
    for k, v in row.items():
        if k.startswith("bitwise"):
            assert v, (k, row)


@pytest.mark.parametrize("cid", am_cases.case_ids("tc"))
def test_conv1d_tc_against_fp64(cid):
    _assert_row(_row("tc", cid))


@pytest.mark.parametrize("cid", am_cases.case_ids("attn"))
def test_attention_tc_against_fp64(cid):
    _assert_row(_row("attn", cid))


def test_bounds_separate_the_modes():
    """The 1xTF32 results of at least one case fail the fp32-accurate bound: the bounds tell the modes apart.  Prints the
    largest err/m per MODE and family."""
    worst = {}
    for fam in ("tc", "attn"):
        rows, _ = _family_rows(fam)
        for r in rows.values():
            if "err_m" in r and np.isfinite(r["err_m"]):
                k = (fam, r["mode"])
                worst[k] = max(worst.get(k, 0.0), r["err_m"])
    print("largest err/m per (family, MODE):", {k: "%.3g (2^%.1f)" % (v, np.log2(v) if v > 0 else -np.inf) for k, v in sorted(worst.items())})
    assert worst[("tc", 0)] > voc_ref.TAU[1] and worst[("attn", 0)] > voc_ref.TAU[1]


# ---- the launch list of one Engine.acoustic call -------------------------------------------------------------------------
POINTS = [(1, (100,)), (3, (9, 23, 14)), (32, None)]      # headline; b3_padded's lengths; 32 utterances of 20-200 phonemes


@pytest.mark.parametrize("invariant", [1, 0], ids=["invariant", "literal"])
@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
def test_launch_list_matches_the_engine(model, lib, dev, prec, invariant):
    """tests/am_plans.engine_launches (the plan-coverage test's list of launches) predicts the number of kernels one
    ev_am_phase1 + ev_am_phase2 call enqueues."""
    from emotivoice_b200 import synth
    eng = model._engine()
    try:
        model.precision = prec
        for B, lens in POINTS:
            lens = list(lens) if lens is not None else synth.corpus_lengths(B)
            bt = {k: v.to(dev) for k, v in synth.make_batch(lens, seed=7 + B).items()}
            torch.cuda.synchronize()
            n0 = lib.ev_launch_count()
            r = eng.acoustic(bt["inputs_ling"], bt["input_lengths"], bt["inputs_speaker"], bt["inputs_style_embedding"],
                             bt["inputs_content_embedding"], invariant)
            n1 = lib.ev_launch_count()
            torch.cuda.synchronize()
            T = bt["inputs_ling"].shape[1]
            want = am_plans.engine_launches(lib, B, T, r["F"], prec, invariant)
            assert n1 - n0 == len(want), (B, T, r["F"], prec, invariant, n1 - n0, len(want))
    finally:
        model.precision = "fp32"
