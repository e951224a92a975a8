"""fp64 references of the vocoder's granule-planar operators and the per-element error bound they are judged by.

Every reference works on one batch item's valid prefix (n rows; rows outside [0, n) are the convolution's zero padding) and on a
window of output rows, so long items can be checked where kernels go wrong -- item ends, tile edges -- without convolving all of
them.  Alongside each result it returns the magnitude m = |bias| + sum |w| |act(x)| (+ |res|, + |prev|, / div): the sum of the
absolute values of every term that enters the output element.  A kernel whose operands carry a relative error u and whose fp32
accumulator adds a few ulps per term is then off by at most ~u * m in that element, whatever the cancellation, so

    |y - y64| <= tau[mode] * m  (+ 2^-9 |y64| where the output is stored in bf16)

holds element by element.  It sees a wrong value where the output is small (zero-padding halos, a ragged last tile), which a
bound relative to max|y64| does not.
"""
import numpy as np
import torch
import torch.nn.functional as F

# mode numbers of the ev_op_*_gp entry points: 0 = 1xTF32, 1 = 3xTF32, 2 = bf16 operands + bf16 storage, 3 = bf16x3
TAU = {0: 2.0 ** -9, 1: 2.0 ** -14, 2: 2.0 ** -6, 3: 2.0 ** -14}
# the bound relative to max|y64| each mode has always been held to
REL_MAX = {0: 3e-3, 1: 5e-5, 2: 1.2e-2, 3: 5e-5}
BF16_OUT = 2.0 ** -9          # one bf16 rounding of the stored output
SLOPE = 0.1                   # LeakyReLU slope of HiFi-GAN's ResBlocks and upsampling (hifigan/models.py:16)


def lrelu(x, slope=SLOPE):
    return torch.where(x >= 0, x, x * slope)


def _padded(xa, r0, r1, pad):
    """Rows [r0 - pad, r1 + pad) of the (n, C) activation xa, zero outside [0, n)."""
    n, C = xa.shape
    out = torch.zeros(r1 - r0 + 2 * pad, C, dtype=xa.dtype)
    a, b = max(r0 - pad, 0), min(r1 + pad, n)
    if b > a:
        out[a - (r0 - pad):b - (r0 - pad)] = xa[a:b]
    return out


def conv_window(xa, w, dil, r0, r1):
    """y[r] = sum_j sum_ci w[j, ci, :] * xa[r + (j - (K-1)/2) * dil, ci] for rows [r0, r1), and the same with |xa|, |w|.
    xa (n, Cin) fp64, already activated; w (K, Cin, Cout).  Returns (y, m), each (r1 - r0, Cout)."""
    K = w.shape[0]
    xs = _padded(xa, r0, r1, (K - 1) // 2 * dil).t().unsqueeze(0)
    wt = w.permute(2, 1, 0).contiguous()                       # (Cout, Cin, K)
    y = F.conv1d(xs, wt, dilation=dil)[0].t()
    m = F.conv1d(xs.abs(), wt.abs(), dilation=dil)[0].t()
    return y, m


def conv_ref(x, w, bias, res, prev, n, r0, r1, dil=1, rate=1, act=True, acc=0, div=1.0):
    """One ev_op_conv1d_gp launch on item rows [r0, r1) of the INPUT resolution.  x (L, Cin), res / prev (L * rate, Cout / rate)
    in the values the kernel reads (bf16-rounded in the bf16 mode).  Returns (y, m) of shape ((r1 - r0) * rate, Cout / rate)."""
    xa = x[:n].double()
    if act:
        xa = lrelu(xa)
    w = w.double()
    y, m = conv_window(xa, w, dil, r0, r1)
    if bias is not None:
        y = y + bias.double()
        m = m + bias.double().abs()
    coutR = w.shape[2] // rate
    y, m = y.reshape(-1, coutR), m.reshape(-1, coutR)           # polyphase: GEMM column group p = output row r * rate + p
    o0, o1 = r0 * rate, r1 * rate
    if res is not None:
        y = y + res[o0:o1].double()
        m = m + res[o0:o1].double().abs()
    if acc:
        y = y + prev[o0:o1].double()
        m = m + prev[o0:o1].double().abs()
        if acc == 2:
            y, m = y / div, m / div
    return y, m


def pair_ref(x, w1, b1, w2, b2, prev, n, r0, r1, dil, acc=0, div=1.0, xt_round=None):
    """One fused ResBlock layer (ev_op_resblock_gp): out = [acc](x + c2(lrelu(c1(lrelu(x), dil)), 1)) on item rows [r0, r1).
    The magnitude carries c1's own error bound into c2: m = |b2| + sum |w2| (|lrelu(xt)| + m1) + |x| (+ |prev|) (/ div), since
    LeakyReLU is 1-Lipschitz.  xt_round rounds the intermediate the way the kernel stores it (bf16 in the bf16 mode)."""
    K = w2.shape[0]
    h2 = (K - 1) // 2
    a, b = max(r0 - h2, 0), min(r1 + h2, n)
    xa = lrelu(x[:n].double())
    xt, m1 = conv_window(xa, w1.double(), dil, a, b)
    xt = xt + b1.double()
    m1 = m1 + b1.double().abs()
    if xt_round is not None:
        xt = xt_round(xt)
    # c2 reads xt rows [r0 - h2, r1 + h2), zero outside [0, n); its magnitude input is |lrelu(xt)| + m1
    full = torch.zeros(n, xt.shape[1], dtype=torch.float64)
    full_m = torch.zeros_like(full)
    full[a:b] = lrelu(xt)
    full_m[a:b] = lrelu(xt).abs() + m1
    y, _ = conv_window(full, w2.double(), 1, r0, r1)
    _, m = conv_window(full_m, w2.double().abs(), 1, r0, r1)
    y = y + b2.double() + x[r0:r1].double()
    m = m + b2.double().abs() + x[r0:r1].double().abs()
    if acc:
        y = y + prev[r0:r1].double()
        m = m + prev[r0:r1].double().abs()
        if acc == 2:
            y, m = y / div, m / div
    return y, m


def post_ref(x, w, bias, n, slope=0.01):
    """conv_post + tanh on one item's valid rows (hifigan/models.py:127-129): x (L, C), w (K, C), bias (1,).  tanh is 1-Lipschitz,
    so the magnitude of the convolution bounds the error of the waveform as well."""
    xa = lrelu(x[:n].double(), slope)
    y, m = conv_window(xa, w.double().unsqueeze(2), 1, 0, n)
    y = torch.tanh(y[:, 0] + bias.double()[0])
    m = m[:, 0] + bias.double().abs()[0]
    return y, m


def bound_excess(y, y64, m, tau, bf16_out=False):
    """Per element (|y - y64| - extra) / m, extra = 2^-9 |y64| for a bf16-stored output; +inf where y is not finite.
    The element passes when this is <= tau."""
    y = y.double()
    err = (y - y64).abs()
    if bf16_out:
        err = err - BF16_OUT * y64.abs()
    r = err / m.clamp_min(1e-300)
    return torch.where(torch.isfinite(y), r, torch.full_like(r, float("inf")))


def check(y, y64, m, mode):
    """-> dict(err_m = max (|y - y64| - extra) / m, rel_max = max|y - y64| / max|y64|, ok)."""
    e = bound_excess(y, y64, m, TAU[mode], bf16_out=(mode == 2))
    err_m = float(e.max()) if e.numel() else 0.0
    d = (y.double() - y64).abs()
    rel = float(d.max() / y64.abs().max().clamp_min(1e-300)) if d.numel() else 0.0
    if not np.isfinite(rel):
        rel = float("inf")
    return dict(err_m=err_m, rel_max=rel, ok=bool(err_m <= TAU[mode] and rel <= REL_MAX[mode]))


def windows(n, tile, width=96, edge=320, n_mid=3):
    """Row windows of an item of n rows to check against the reference: the first and last `edge` rows and +-width/2 rows
    around the tile edges k * tile for the first, a few middle and the last k.  Merged, sorted, within [0, n)."""
    ws = [(0, min(n, edge)), (max(0, n - edge), n)]
    ks = list(range(1, (n - 1) // tile + 1)) if tile > 0 else []
    if ks:
        pick = sorted({ks[0], ks[-1]} | {ks[i * len(ks) // (n_mid + 1)] for i in range(1, n_mid + 1)})
        for k in pick:
            ws.append((max(0, k * tile - width // 2), min(n, k * tile + width // 2)))
    ws.sort()
    out = []
    for a, b in ws:
        if b <= a:
            continue
        if out and a <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], b))
        else:
            out.append((a, b))
    return out
