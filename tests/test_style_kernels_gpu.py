"""The style encoder's tensor-core GEMMs against fp64, at every layer shape, kernel MODE, K-split factor and tile plan
ev_style_forward issues for BERT-base and the small model, and at token counts on the tile edges; and the whole BERT-base
forward of a ragged batch against its items' batch-1 calls.

Operator level (cases and child process: the "style" family of tests/am_cases.py; reference and bound: tests/am_ref.py; launch
list: tests/style_plans.py).  The family runs once in its own process under a timeout, as in tests/test_am_kernels_gpu.py, and
no case is ever run twice.  Every valid output element must satisfy |y - y64| <= tau[MODE] * m, with tau = 2^-14 (3xTF32,
"fp32") and 2^-9 (1xTF32, "tf32"), and the bound relative to max|y64| of each mode.  Rows past each item are NaN on input and
must come out as exact zeros.  Bitwise: two runs; each edge-length item of a ragged batch against its own batch-1 launch (at
another N tile width, for all but the widest layers).

Largest err/m measured on an H100 80GB HBM3 (132 SMs, 400 W power limit), tau = 2^-14 for MODE 1 and 2^-9 for MODE 0.  The
longest fp32 chain is BERT-base's 3xTF32 ffn2 slice of 768 products, <= 767 * 2^-24 ~ 2^-14.4 of m in the worst case:
                      qkv       wo        ffn1      ffn2
    base    MODE 1    2^-20.0   2^-20.0   2^-20.3   2^-19.9
            MODE 0    2^-13.5   2^-13.6   2^-13.5   2^-14.1
    small   MODE 1    2^-20.8   2^-21.0   2^-21.1   2^-21.0
            MODE 0    2^-12.8   2^-12.9   2^-13.0   2^-13.6
The child process took 13 s for its 128 cases, fp64 references on the host's 16 CPU threads included; the whole file about 25 s.
"""
import numpy as np
import pytest
import torch

import am_cases
import style_plans
import voc_ref
from test_am_kernels_gpu import _assert_row, _family_rows
from test_zz_late_round1_gpu import STYLE_OUTS, _style_model

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cid", am_cases.case_ids("style"))
def test_style_gemm_against_fp64(cid):
    rows, tail = _family_rows("style")
    assert cid in rows, "no result row for %s: %s" % (cid, tail)
    row = rows[cid]
    _assert_row(row)
    want = {"bound_ok", "pad_zero", "bitwise_two_runs"} | ({"bitwise_item_vs_batch1"} if row["B"] > 1 else set())
    assert want <= set(row), row


def test_bounds_separate_the_modes():
    """The 1xTF32 results of at least one case fail the 3xTF32 bound.  Prints the largest err/m per (config, kind, MODE)."""
    rows, _ = _family_rows("style")
    worst = {}
    for r in rows.values():
        if "err_m" in r and np.isfinite(r["err_m"]):
            k = (r["kind"], r["mode"])
            worst[k] = max(worst.get(k, 0.0), r["err_m"])
    print("largest err/m per (config:kind, MODE):",
          {k: "%.3g (2^%.1f)" % (v, np.log2(v) if v > 0 else -np.inf) for k, v in sorted(worst.items())})
    assert any(v > voc_ref.TAU[1] for (_, mode), v in worst.items() if mode == 0)


# ---- the launch list of one ev_style_forward call -------------------------------------------------------------------------
POINTS = ((1, 20), (3, 129), (32, 512))         # token counts above a configuration's max_position are clamped to it


def _forward(lib, eng, B, N, heads, seed=0):
    """One ev_style_forward of B items of N tokens (the first item full, the others shorter); returns the launches it enqueued."""
    dev = eng.device
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, int(eng.cfg.vocab_size), (B, N), generator=g).to(dev)
    tts = torch.randint(0, int(eng.cfg.type_vocab), (B, N), generator=g).to(dev)
    lens = torch.randint(1, N + 1, (B,), generator=g)
    lens[0] = N
    lens = lens.to(dev)
    pooled = torch.empty(B, int(eng.cfg.hidden), device=dev)
    out_heads = torch.empty(B, eng.n_head_out, device=dev) if heads else None
    n = int(lib.ev_style_workspace_bytes(eng.handle, B, N))
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    n0 = lib.ev_launch_count()
    rc = lib.ev_style_forward(eng.handle, ids.data_ptr(), tts.data_ptr(), lens.data_ptr(), B, N, pooled.data_ptr(),
                              None if out_heads is None else out_heads.data_ptr(), ws.data_ptr(), n,
                              torch.cuda.current_stream(dev).cuda_stream)
    n1 = lib.ev_launch_count()
    torch.cuda.synchronize()
    assert rc == 0, lib.ev_last_error().decode(errors="replace")
    return n1 - n0


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("cfg", style_plans.CONFIGS)
def test_launch_list_matches_the_engine(lib, dev, cfg, prec):
    """tests/style_plans.style_launches (the style plan-coverage test's list of launches) predicts the number of kernels one
    ev_style_forward call enqueues, with and without the heads."""
    m = _style_model(cfg == "small", dev)
    eng = m._engine()
    nmax = int(eng.cfg.max_position)
    try:
        m.precision = prec
        for B, N in POINTS:
            N = min(N, nmax)
            for heads in (True, False):
                got = _forward(lib, eng, B, N, heads, seed=B + N)
                want = style_plans.style_launches(lib, cfg, B, N, prec, heads=heads)
                assert got == len(want), (cfg, prec, B, N, heads, got, len(want))
    finally:
        m.precision = "fp32"


# ---- the whole BERT-base forward: a ragged batch == its items alone ------------------------------------------------------
def test_base_ragged_batch_equals_its_batch1_calls(lib, dev):
    """frontdoor.PromptEmbeddingCache sends every uncached text through the encoder as one right-padded batch and promises the
    result is bitwise what a batch-1 call gives.  12 items padded to 512 tokens, on and next to the 128-row tile edges, the
    padding filled with random in-range ids and token types (what a caller's buffer may hold, not [PAD]): pooled_output and
    the four heads of every item equal its own batch-1 call bitwise, in "fp32" and in "tf32"."""
    m = _style_model(False, dev)
    sc = m.arch
    g = torch.Generator().manual_seed(2024)
    lens = [512, 1, 2, 127, 128, 129, 255, 256, 257] + torch.randint(3, 512, (3,), generator=g).tolist()
    B, N = len(lens), 512
    ids = torch.randint(0, int(sc.vocab_size), (B, N), generator=g)
    tts = torch.randint(0, int(sc.type_vocab_size), (B, N), generator=g)
    mask = (torch.arange(N)[None, :] < torch.tensor(lens)[:, None]).to(torch.int64)
    try:
        for prec in ("fp32", "tf32"):
            m.precision = prec
            full = m(input_ids=ids.to(dev), token_type_ids=tts.to(dev), attention_mask=mask.to(dev))
            for b, n in enumerate(lens):
                one = m(input_ids=ids[b:b + 1, :n].to(dev), token_type_ids=tts[b:b + 1, :n].to(dev),
                        attention_mask=mask[b:b + 1, :n].to(dev))
                for k in STYLE_OUTS:
                    assert torch.equal(one[k][0], full[k][b]), (prec, b, n, k)
            assert bool(torch.isfinite(full["pooled_output"]).all())
    finally:
        m.precision = "fp32"
