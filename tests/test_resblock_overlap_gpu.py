"""The fused ResBlock kernel's cross-tile path on the GPU: bitwise equal to the two conv1d_gp launches it replaces.

Each CTA of `resblock_gp_kernel` stores epi2 of its tile i under c1 of its next active tile, and the last epi2 after its last
tile (DESIGN.md §3.2).  The cases below make CTAs take one, two and many tiles, end on a tile of every member of a grouped
launch, skip the inactive tiles of a ragged batch (items of one unit, rows past each length NaN on input), and run the
accumulate modes (ACC_ADD_DIV's epilogue waits for c1 instead).  Every case compares the fused output bitwise with the two
conv1d_gp launches (solo) or with the members' own fused launches (grouped), in all four modes.  The cases run in a child process
under a timeout, as in tests/test_voc_kernels_gpu.py: a pipeline that deadlocks ends the child, not the suite.

    python tests/test_resblock_overlap_gpu.py      (the child: one JSON row per case)
"""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

# name, B, L, C, K (or Ks of a grouped launch), dil, acc, lens in units of `mul` rows (None: full length)
SOLO = [("one_tile_per_cta", 1, 5000, 64, 3, 1, 0, None),
        ("two_tiles_per_cta", 1, 50800, 64, 7, 3, 0, None),
        ("many_tiles_C32", 3, 70000, 32, 11, 5, 1, (70000, 1, 40000)),
        ("many_tiles_C64_div", 4, 40000, 64, 11, 5, 2, (40000, 9000, 1, 25000)),
        ("ragged_C128", 8, 20000, 128, 3, 1, 0, (20000, 1, 1, 15000, 1, 7, 1, 19999))]
GROUPED = [("grouped_C64", 1, 65536, 64, (3, 7, 11), 3, None),
           ("grouped_C32", 1, 131072, 32, (11, 3, 7), 5, None),
           ("grouped_C32_ragged", 3, 20000, 32, (3, 7, 11), 1, (20000, 1, 9001))]
MODES = (0, 1, 2, 3)


def _child():
    sys.path.insert(0, HERE)
    import math
    import ctypes
    import torch
    import voc_cases as vc
    lib = vc._setup()
    from emotivoice_b200 import layout
    R = vc.Runner(lib)
    dev = R.dev
    for name, B, L, C, K, dil, accm, lens in SOLO:
        for mode in MODES:
            g = torch.Generator().manual_seed(7)
            lens = lens or (L,) * B
            valid = [min(L, v) for v in lens]
            bf = mode == 2
            x = vc._nan_past(torch.randn(B, L, C, generator=g), valid)
            w1 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
            w2 = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
            b1, b2 = torch.randn(C, generator=g), torch.randn(C, generator=g)
            init = vc._nan_past(torch.randn(B, L, C, generator=g) if accm else torch.full((B, L, C), float("nan")), valid)
            xg = layout.to_gp(x, bf).to(dev)
            w1d, w2d, b1d, b2d = vc._pack(mode)(w1).to(dev), vc._pack(mode)(w2).to(dev), b1.to(dev), b2.to(dev)
            before = layout.to_gp(init, bf)
            out, ref, xt = before.to(dev), before.to(dev), torch.full_like(xg, float("nan"))
            lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
            rc = lib.ev_op_resblock_gp(R.ptr(xg), R.ptr(w1d), R.ptr(b1d), R.ptr(w2d), R.ptr(b2d), mode, R.ptr(out), B, L, C, K, dil, R.ptr(lens_d), 1,
                                       accm, 3.0, R.st)
            rc1 = vc._conv_launch(R, mode, xg, w1d, b1d, None, xt, B, L, C, K, dil, lens_d, 1)
            rc2 = vc._conv_launch(R, mode, xt, w2d, b2d, xg, ref, B, L, C, K, 1, lens_d, 1, accm, 3.0)
            torch.cuda.synchronize()
            got = out.cpu()
            ok = rc == 0 and rc1 == 0 and rc2 == 0 and vc._gp_valid_equal(got, ref.cpu(), valid) and vc._pad_ok(got, before, valid)
            print(json.dumps(dict(case="%s-m%d" % (name, mode), ok=bool(ok), rc=[rc, rc1, rc2], err=R.err() if rc else "")), flush=True)
    for name, B, L, C, Ks, dil, lens in GROUPED:
        for mode in MODES:
            g = torch.Generator().manual_seed(11)
            n = len(Ks)
            lens = lens or (L,) * B
            valid = [min(L, v) for v in lens]
            bf = mode == 2
            xg = [layout.to_gp(vc._nan_past(torch.randn(B, L, C, generator=g), valid), bf).to(dev) for _ in Ks]
            w1d = [vc._pack(mode)(torch.randn(K, C, C, generator=g) / math.sqrt(C * K)).to(dev) for K in Ks]
            w2d = [vc._pack(mode)(torch.randn(K, C, C, generator=g) / math.sqrt(C * K)).to(dev) for K in Ks]
            b1d = [torch.randn(C, generator=g).to(dev) for _ in Ks]
            b2d = [torch.randn(C, generator=g).to(dev) for _ in Ks]
            before = layout.to_gp(torch.full((B, L, C), float("nan")), bf)
            grp, solo = [before.to(dev) for _ in Ks], [before.to(dev) for _ in Ks]
            lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
            rcs = [lib.ev_op_resblock_gp(R.ptr(xg[i]), R.ptr(w1d[i]), R.ptr(b1d[i]), R.ptr(w2d[i]), R.ptr(b2d[i]), mode, R.ptr(solo[i]), B, L, C, Ks[i], dil,
                                         R.ptr(lens_d), 1, 0, 1.0, R.st) for i in range(n)]
            IA = ctypes.c_int * n
            rc = lib.ev_op_resblock_gp_group(n, vc._tab(R, xg), vc._tab(R, w1d), vc._tab(R, b1d), vc._tab(R, w2d), vc._tab(R, b2d), mode, vc._tab(R, grp),
                                             B, L, C, IA(*Ks), IA(*([dil] * n)), R.ptr(lens_d), 1, R.st)
            torch.cuda.synchronize()
            ok = rc == 0 and not any(rcs)
            for i in range(n):
                got = grp[i].cpu()
                ok = ok and vc._gp_valid_equal(got, solo[i].cpu(), valid) and vc._pad_ok(got, before, valid)
            print(json.dumps(dict(case="%s-m%d" % (name, mode), ok=bool(ok), rc=[rc] + rcs, err=R.err() if rc else "")), flush=True)


def case_ids():
    return ["%s-m%d" % (c[0], m) for c in SOLO + GROUPED for m in MODES]


_ROWS = {}


def _rows():
    if not _ROWS:
        p = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, timeout=900)
        for line in p.stdout.splitlines():
            if line.startswith("{"):
                r = json.loads(line)
                _ROWS[r["case"]] = r
        _ROWS["__stderr__"] = p.stderr[-3000:]
    return _ROWS


@pytest.mark.gpu
@pytest.mark.parametrize("cid", case_ids())
def test_fused_bitwise_across_tiles(cid):
    rows = _rows()
    assert cid in rows, "case did not run:\n" + rows["__stderr__"]
    assert rows[cid]["ok"], rows[cid]


if __name__ == "__main__":
    _child()
