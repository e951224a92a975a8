"""fp64 numpy restatement of ``emotivoice_b200.evaluate`` / ``ev_eval_compare``: cepstra of log-mels, the local distance, dynamic
time warping (DTW) with its tie order, the backtracked path and the statistics along it.

Every sum runs in the order the definitions give, one rounded operation at a time (numpy's elementwise float64 operations are
IEEE with no fused multiply-add), so the cepstra, distances, DTW costs and paths are bitwise those of the kernels.  The last
steps (log2 of an F0 ratio, the final scale of mcd) go through libm and agree to an ulp or two.
"""
import math

import numpy as np

N_MELS, N_CEPS = 80, 24
MCD_K = 10.0 * math.sqrt(2.0) / math.log(10.0)          # dB per unit of cepstral distance
START, DIAG, UP, LEFT = 3, 0, 1, 2                        # predecessor codes


def cos_table():
    """(24, 80) float64: row k - 1 holds cos(pi k (m + 1/2) / 80), m = 0..79."""
    k = np.arange(1, N_CEPS + 1, dtype=np.float64)[:, None]
    m = np.arange(N_MELS, dtype=np.float64)[None, :]
    return np.cos(np.pi * k * (m + 0.5) / N_MELS)


def cepstra(logmel, table=None):
    """(80, N) log-mel -> (N, 24) float64: c_k[f] = (sum over ascending m of fp64(L[m, f]) * T[k, m]) / 80."""
    L = np.asarray(logmel, dtype=np.float64)
    T = cos_table() if table is None else np.asarray(table, dtype=np.float64)
    acc = np.zeros((N_CEPS, L.shape[1]))
    for m in range(N_MELS):                                  # elementwise, so numpy's pairwise summation never enters
        acc = acc + T[:, m:m + 1] * L[m][None, :]
    return (acc / float(N_MELS)).T.copy()


def distances(ca, cb):
    """(N, 24), (M, 24) cepstra -> (N, M) d(i, j) = sqrt(sum over ascending k of (c_k[i] - c'_k[j])^2)."""
    acc = np.zeros((ca.shape[0], cb.shape[0]))
    for k in range(N_CEPS):
        df = ca[:, k][:, None] - cb[:, k][None, :]
        acc = acc + df * df
    return np.sqrt(acc)


def dtw(d):
    """(N, M) local distances -> (D (N, M) accumulated costs, codes (N, M) int8), computed per anti-diagonal.  D(0,0) = d(0,0);
    D(i,j) = d(i,j) + min over the existing predecessors, ties to the first of (i-1, j-1), (i-1, j), (i, j-1)."""
    N, M = d.shape
    D = np.full((N, M), np.nan)
    code = np.full((N, M), -1, np.int8)
    D[0, 0], code[0, 0] = d[0, 0], START
    for t in range(1, N + M - 1):
        i = np.arange(max(0, t - M + 1), min(t, N - 1) + 1)
        j = t - i
        best = np.full(i.shape, np.inf)
        c = np.full(i.shape, -1, np.int8)
        inner = (i > 0) & (j > 0)
        best[inner] = D[i[inner] - 1, j[inner] - 1]
        c[inner] = DIAG
        up = i > 0
        v = np.full(i.shape, np.inf)
        v[up] = D[i[up] - 1, j[up]]
        take = up & ((c < 0) | (v < best))
        best[take], c[take] = v[take], UP
        left = j > 0
        v = np.full(i.shape, np.inf)
        v[left] = D[i[left], j[left] - 1]
        take = left & ((c < 0) | (v < best))
        best[take], c[take] = v[take], LEFT
        D[i, j] = d[i, j] + best
        code[i, j] = c
    return D, code


def backtrack(code):
    """-> (P, 2) int32 path from (0,0) to (N-1, M-1)."""
    i, j = code.shape[0] - 1, code.shape[1] - 1
    path = [(i, j)]
    while code[i, j] != START:
        c = code[i, j]
        if c == DIAG:
            i, j = i - 1, j - 1
        elif c == UP:
            i -= 1
        else:
            j -= 1
        path.append((i, j))
    return np.array(path[::-1], dtype=np.int32)


def statistics(d, path, f0_syn, f0_ref):
    """Sums along the path in path order from (0,0) -> dict of mcd, f0_rmse, vuv_error, voiced_pairs, path_length."""
    P = len(path)
    s = 0.0
    e, voiced, mismatch = 0.0, 0, 0
    for i, j in path:
        s = s + float(d[i, j])
        a, r = float(f0_syn[i]), float(f0_ref[j])
        va, vr = a > 0.0, r > 0.0
        mismatch += va != vr
        if va and vr:
            cents = 1200.0 * math.log2(a / r)
            e = e + cents * cents
            voiced += 1
    return dict(mcd=MCD_K * (s / P), f0_rmse=math.sqrt(e / voiced) if voiced else math.nan, vuv_error=mismatch / P,
                voiced_pairs=voiced, path_length=P, cost=s)


def compare(logmel_syn, f0_syn, logmel_ref, f0_ref, table=None):
    """One pair from its (80, N), (80, M) log-mels and (N,), (M,) F0 tracks (0 unvoiced) -> statistics(...) plus "path" and
    "D" (the accumulated cost at (N-1, M-1))."""
    d = distances(cepstra(logmel_syn, table), cepstra(logmel_ref, table))
    D, code = dtw(d)
    path = backtrack(code)
    out = statistics(d, path, np.asarray(f0_syn, np.float64), np.asarray(f0_ref, np.float64))
    out.update(path=path, D=float(D[-1, -1]))
    return out
