"""The comparison of syntheses with recordings on the host (no GPU): the fp64 oracle's DTW against a textbook double-loop DP
and, on small grids, against every monotone path; known answers (identical and repeated sequences, a level offset); and the
argument errors ``evaluate.compare`` raises before it touches a device."""
import math

import numpy as np
import pytest
import torch

from emotivoice_b200 import evaluate, feats
from oracle import eval_oracle as O


def textbook_dtw(d):
    """Row by row double loop: the cost and the path, ties to the diagonal, then (i-1, j), then (i, j-1)."""
    N, M = d.shape
    D = np.zeros((N, M))
    prev = {}
    for i in range(N):
        for j in range(M):
            if i == 0 and j == 0:
                D[i, j] = d[i, j]
                continue
            cands = []
            if i > 0 and j > 0:
                cands.append((D[i - 1, j - 1], (i - 1, j - 1)))
            if i > 0:
                cands.append((D[i - 1, j], (i - 1, j)))
            if j > 0:
                cands.append((D[i, j - 1], (i, j - 1)))
            best = cands[0]
            for c in cands[1:]:
                if c[0] < best[0]:
                    best = c
            D[i, j] = d[i, j] + best[0]
            prev[(i, j)] = best[1]
    path, cell = [(N - 1, M - 1)], (N - 1, M - 1)
    while cell != (0, 0):
        cell = prev[cell]
        path.append(cell)
    return D[-1, -1], np.array(path[::-1], np.int32)


def all_monotone_paths(N, M):
    """Every path from (0,0) to (N-1, M-1) with steps (1,1), (1,0), (0,1)."""
    def walk(i, j):
        if (i, j) == (N - 1, M - 1):
            yield [(i, j)]
            return
        for di, dj in ((1, 1), (1, 0), (0, 1)):
            if i + di < N and j + dj < M:
                for rest in walk(i + di, j + dj):
                    yield [(i, j)] + rest
    return walk(0, 0)


@pytest.mark.parametrize("seed", range(40))
def test_oracle_dtw_equals_the_textbook_dp(seed):
    rng = np.random.default_rng(seed)
    N, M = (int(v) for v in rng.integers(1, 40, size=2))
    d = rng.random((N, M))
    if seed % 4 == 0:
        d = np.round(d * 3) / 3                   # many ties
    D, code = O.dtw(d)
    path = O.backtrack(code)
    cost, ref_path = textbook_dtw(d)
    assert D[-1, -1] == cost
    assert np.array_equal(path, ref_path)
    assert max(N, M) <= len(path) <= N + M - 1
    s = 0.0
    for i, j in path:
        s = s + d[i, j]
    assert s == D[-1, -1]                         # the path-order sum is the DTW cost, bit for bit


@pytest.mark.parametrize("N,M", [(1, 1), (1, 5), (4, 1), (3, 3), (4, 6), (6, 6), (5, 2)])
def test_oracle_cost_is_the_minimum_over_every_monotone_path(N, M):
    rng = np.random.default_rng(N * 10 + M)
    d = rng.random((N, M))
    best = min(sum(d[i, j] for i, j in p) for p in all_monotone_paths(N, M))
    D, _ = O.dtw(d)
    assert abs(D[-1, -1] - best) <= 1e-12 * best


def test_identical_sequences_give_the_diagonal_and_zero():
    rng = np.random.default_rng(3)
    L = rng.normal(-4.0, 2.0, size=(80, 57))
    f0 = np.where(rng.random(57) > 0.3, rng.uniform(80, 300, 57), 0.0)
    r = O.compare(L, f0, L, f0)
    assert np.array_equal(r["path"], np.stack([np.arange(57)] * 2, axis=1))
    assert r["mcd"] == 0.0 and r["vuv_error"] == 0.0 and r["f0_rmse"] == 0.0
    assert r["voiced_pairs"] == int((f0 > 0).sum())


def test_repeated_frames_give_zero_and_follow_the_repeats():
    rng = np.random.default_rng(4)
    L = rng.normal(-4.0, 2.0, size=(80, 20))
    reps = rng.integers(1, 4, size=20)
    idx = np.repeat(np.arange(20), reps)
    r = O.compare(L, np.zeros(20), L[:, idx], np.zeros(len(idx)))
    assert r["mcd"] == 0.0
    assert np.array_equal(r["path"], np.stack([idx, np.arange(len(idx))], axis=1))
    assert math.isnan(r["f0_rmse"]) and r["voiced_pairs"] == 0


def test_a_level_offset_moves_only_c0():
    rng = np.random.default_rng(5)
    L = rng.normal(-4.0, 2.0, size=(80, 30))
    for off in (-3.0, 0.7, 5.0):
        assert np.abs(O.cepstra(L + off) - O.cepstra(L)).max() <= 1e-13


def test_the_product_and_the_oracle_build_the_same_table():
    assert np.array_equal(evaluate.cos_table().view(np.int64), O.cos_table().view(np.int64))
    assert evaluate.MIN_SAMPLES == feats.pitch_min_samples(16000) == 641
    assert evaluate.MAX_SAMPLES == 4096 * 256 - 1


class _FakeCuda(torch.Tensor):
    """A CPU tensor that claims to be on the GPU, so the checks after the device check run without one."""
    @property
    def is_cuda(self):
        return True


def _fake(B, L):
    return torch.zeros((B, L), dtype=torch.float32).as_subclass(_FakeCuda)


def test_argument_errors_need_no_gpu():
    cpu = torch.zeros((2, 16000))
    for syn, ref in ((cpu, cpu), (cpu.double(), cpu), (cpu[0], cpu), (cpu, cpu.half())):
        with pytest.raises(ValueError):
            evaluate.compare(syn, ref)
    s, r = _fake(2, 16000), _fake(2, 20000)
    bad = [dict(sample_rate=3000), dict(sample_rate=16001), dict(sample_rate=16000.5), dict(sample_rate="16k"),
           dict(syn_lengths=[640, 16000]), dict(ref_lengths=[16000, 20001]), dict(syn_lengths=[1000]),
           dict(syn_lengths=[1000.0, 2000]), dict(syn_lengths=[True, 2000]), dict(return_path=1),
           dict(sample_rate=48000, syn_lengths=[1920, 3000])]
    for kw in bad:
        with pytest.raises(ValueError):
            evaluate.compare(s, r, **kw)
    with pytest.raises(ValueError):
        evaluate.compare(_fake(1, 4096 * 256), _fake(1, 16000))             # 4097 frames
    with pytest.raises(ValueError):
        evaluate.compare(_fake(2, 16000), _fake(3, 16000))
    with pytest.raises(ValueError):
        evaluate.compare(_fake(2, 16000), _fake(2, 16000), ref_lengths=torch.tensor([1000, 1000], device="meta"))
