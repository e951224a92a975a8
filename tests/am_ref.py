"""fp64 references of the acoustic model's tensor-core operators (conv1d_tc + splitk_reduce, attention_tc) and the per-element
magnitudes they are judged by.

Like tests/voc_ref.py, every reference returns, next to each output element y64, a magnitude m such that a kernel whose
operands carry a relative error u and whose fp32 accumulators add a few ulps per term is off by at most ~u * m there, whatever
the cancellation.  The element passes when |y - y64| <= tau[MODE] * m (voc_ref.TAU; voc_ref.bound_excess), and the whole result
must also meet the bound relative to max|y64| each mode has always been held to.

* Convolution / linear layer (one item's valid rows, rows outside [0, n) are the zero padding):
      y = act(bias[b] + sum_j sum_ci w[j, ci, :] x[r + j - (K-1)/2, ci]) (+ res),   m = L_act (|bias[b]| + sum |w| |x|) (+ |res|)
  with L_act the activation's Lipschitz constant: 1 for none / ReLU, 1.13 for the exact (erf) GELU (max |gelu'(x)| = 1.1289 at
  x = +-sqrt(2)), so an error of the pre-activation sum stays within L_act times its own bound after the activation.
* Attention (encoder.py:84-109), per query row i and channel d of a head, over the keys j < klen:
      o = sum_j p_j v_j,  p = softmax(s),  s_j = q . k_j / sqrt(d_k)
      m = sum_j p_j |v_j| + sum_j p_j a_j |v_j - o|,   a_j = sum_d |q_d k_jd| / sqrt(d_k)
  The first term is the product P V's own magnitude.  The second carries the operand error of the scores through the softmax:
  an error e_j = u a_j of score j moves o by sum_j p_j e_j (v_j - o) (d o / d s_j = p_j (v_j - o)), which for large scores
  (the lazily rescaled online softmax with tf32 operands) is far more than u sum p |v|.
"""
import math

import torch
import torch.nn.functional as F

import voc_ref

TAU, REL_MAX = voc_ref.TAU, voc_ref.REL_MAX
GELU_LIP = 1.13
ACT_NONE, ACT_RELU, ACT_GELU = 0, 2, 3
# attention: the bounds relative to max|y64| of the 3xTF32 / 1xTF32 modes; with scores of ~100 (the lazily rescaled softmax) the
# tf32 one of test_attention_tc_lazy_rescale_path
ATTN_REL_MAX = {1: REL_MAX[1], 0: REL_MAX[0]}
ATTN_REL_MAX_LARGE_SCORES = {1: REL_MAX[1], 0: 2e-2}


def conv_ref(x, w, bias, res, n, out_act=ACT_NONE, r0=0, r1=None):
    """One ev_op_conv1d_tc launch on one item's rows [r0, r1) of its n valid rows: x (L, Cin), w (K, Cin, Cout), bias (Cout,)
    -- the item's own row where the engine passes a per-item bias --, res (L, Cout) or None.  Returns (y, m), each (r1 - r0, Cout)."""
    r1 = n if r1 is None else r1
    y, m = voc_ref.conv_window(x[:n].double(), w.double(), 1, r0, r1)
    if bias is not None:
        y = y + bias.double()
        m = m + bias.double().abs()
    if out_act == ACT_RELU:
        y = torch.relu(y)
    elif out_act == ACT_GELU:
        y = F.gelu(y)
        m = m * GELU_LIP
    if res is not None:
        y = y + res[r0:r1].double()
        m = m + res[r0:r1].double().abs()
    return y, m


def attn_ref(qkv, klen, heads, rows=None, score_term=True, chunk=16):
    """encoder.py:84-109 for one item: qkv (L, 3H) with the keys / values j < klen, queries at `rows` (default: all of
    [0, klen)).  Returns (o, m), each (len(rows), H).  score_term=False leaves the softmax term out of m (for the test
    that shows it is needed)."""
    L, H3 = qkv.shape
    H = H3 // 3
    dk = H // heads
    rows = torch.arange(klen) if rows is None else torch.as_tensor(rows)
    t = qkv.double()
    q = t[rows, :H].reshape(-1, heads, dk).transpose(0, 1)              # (h, nq, dk)
    k = t[:klen, H:2 * H].reshape(klen, heads, dk).transpose(0, 1)      # (h, n, dk)
    v = t[:klen, 2 * H:].reshape(klen, heads, dk).transpose(0, 1)
    sc = 1.0 / math.sqrt(dk)
    p = torch.softmax(q @ k.transpose(1, 2) * sc, -1)                   # (h, nq, n)
    o = p @ v
    m = p @ v.abs()
    if score_term:
        w = p * (q.abs() @ k.abs().transpose(1, 2) * sc)                # p_j a_j
        extra = torch.empty_like(m)
        for i0 in range(0, q.shape[1], chunk):
            i1 = min(i0 + chunk, q.shape[1])
            dev = (v[:, None, :, :] - o[:, i0:i1, None, :]).abs()        # (h, c, n, dk)
            extra[:, i0:i1] = (w[:, i0:i1, :, None] * dev).sum(2)
        m = m + extra
    return o.transpose(0, 1).reshape(-1, H), m.transpose(0, 1).reshape(-1, H)


def check(y, y64, m, mode, rel_max=None):
    """-> dict(err_m = max |y - y64| / m (inf where y is not finite), rel_max = max|y - y64| / max|y64|, ok).  The acoustic
    model's tensor-core outputs are fp32 in every mode, so no storage rounding is added."""
    e = voc_ref.bound_excess(y, y64, m, TAU[mode])
    err_m = float(e.max()) if e.numel() else 0.0
    d = (y.double() - y64).abs()
    rel = float(d.max() / y64.abs().max().clamp_min(1e-300)) if d.numel() else 0.0
    if not math.isfinite(rel):
        rel = float("inf")
    lim = REL_MAX[mode] if rel_max is None else rel_max
    return dict(err_m=err_m, rel_max=rel, ok=bool(err_m <= TAU[mode] and rel <= lim))
