"""Per-kernel parity: every CUDA operator behind the C ABI against the matching piece of the
oracle / a plain PyTorch fp32 CPU reference on seeded tensors.  Tolerances are fp32
round-off level (the kernels accumulate in fp32 FFMA, like the CPU reference does in a
different order): |err| <= 2e-5 * max|ref| unless stated."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_max
from emotivoice_b200 import _abi, packing
from oracle import jets_oracle as O

pytestmark = pytest.mark.gpu
TOL = 2e-5


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def run_conv(lib, x_tm, w_kio, bias, res, out_init, K, dil, lens, lens_mul, in_act, in_slope, out_act, acc, div, bias_bs=0):
    B, L, Cin = x_tm.shape
    Cout = w_kio.shape[2]
    out = out_init.clone() if out_init is not None else torch.full((B, L, Cout), float("nan"), device=x_tm.device)
    _abi.check(lib.ev_op_conv1d(_ptr(x_tm), _ptr(w_kio), _ptr(bias), bias_bs, _ptr(res), _ptr(out), B, L, Cin, Cout, K, dil,
                                _ptr(lens), lens_mul, in_act, in_slope, out_act, acc, div, _stream()))
    torch.cuda.synchronize()
    return out


CONV_CASES = [
    # B, L, Cin, Cout, K, dil   (tile variants: Cout<=32, <=64, small, big)
    (1, 300, 32, 32, 11, 5),
    (2, 517, 64, 64, 7, 3),
    (1, 100, 384, 1152, 1, 1),
    (1, 260, 384, 1536, 3, 1),
    (2, 130, 1536, 384, 3, 1),
    (1, 70, 80, 512, 7, 1),
    (3, 700, 128, 128, 3, 1),
    (2, 2100, 256, 256, 11, 1),
    (1, 537, 384, 80, 1, 1),
    (1, 5000, 32, 32, 3, 3),
    (40, 150, 64, 64, 3, 1),
]


@pytest.mark.parametrize("B,L,Cin,Cout,K,dil", CONV_CASES)
def test_conv1d_matches_torch(lib, dev, B, L, Cin, Cout, K, dil):
    g = torch.Generator().manual_seed(B * 1000 + L + Cin + Cout + K)
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g)
    ref = F.conv1d(F.leaky_relu(x, 0.1), w, b, padding=(K - 1) // 2 * dil, dilation=dil).transpose(1, 2)
    out = run_conv(lib, x.transpose(1, 2).contiguous().to(dev), packing._conv_w(w).to(dev), b.to(dev), None, None,
                   K, dil, None, 1, _abi.ACT_LRELU, 0.1, _abi.ACT_NONE, _abi.ACC_STORE, 1.0)
    assert rel_max(out.cpu(), ref) <= TOL


@pytest.mark.parametrize("out_act", [_abi.ACT_GELU, _abi.ACT_RELU, _abi.ACT_TANH])
def test_conv1d_epilogues(lib, dev, out_act):
    g = torch.Generator().manual_seed(5 + out_act)
    B, L, Cin, Cout, K = 2, 77, 48, 96, 3
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g)
    res = torch.randn(B, L, Cout, generator=g)
    prev = torch.randn(B, L, Cout, generator=g)
    y = F.conv1d(x, w, b, padding=1)
    y = {_abi.ACT_GELU: F.gelu, _abi.ACT_RELU: F.relu, _abi.ACT_TANH: torch.tanh}[out_act](y).transpose(1, 2)
    ref = (prev + (y + res)) / 3.0
    out = run_conv(lib, x.transpose(1, 2).contiguous().to(dev), packing._conv_w(w).to(dev), b.to(dev), res.to(dev),
                   prev.to(dev), K, 1, None, 1, _abi.ACT_NONE, 0.0, out_act, _abi.ACC_ADD_DIV, 3.0)
    assert rel_max(out.cpu(), ref) <= TOL
    # in-place residual (out aliases res), as the engine runs x += f(x)
    xt = x.transpose(1, 2).contiguous().to(dev)
    buf = res.to(dev).clone()
    wd, bd = packing._conv_w(w).to(dev), b.to(dev)
    _abi.check(lib.ev_op_conv1d(xt.data_ptr(), wd.data_ptr(), bd.data_ptr(), 0,
                                buf.data_ptr(), buf.data_ptr(), B, L, Cin, Cout, K, 1, None, 1, 0, 0.0, out_act, 0, 1.0,
                                _stream()))
    torch.cuda.synchronize()
    assert rel_max(buf.cpu(), y + res) <= TOL


def test_conv1d_ragged_lengths_equal_b1(lib, dev):
    """rows >= lens[b]*mul read as zero padding and are stored as zeros: item b of a padded
    batch equals the B=1 convolution of its valid prefix, BITWISE."""
    g = torch.Generator().manual_seed(11)
    B, L, C, K, dil, mul = 3, 96 * 4, 64, 7, 3, 4
    lens = torch.tensor([96, 17, 50], dtype=torch.int32)
    x = torch.randn(B, L, C, generator=g).to(dev)
    w = (torch.randn(K, C, C, generator=g) / math.sqrt(C * K)).to(dev)
    b = torch.randn(C, generator=g).to(dev)
    out = run_conv(lib, x, w, b, None, None, K, dil, lens.to(dev), mul, _abi.ACT_LRELU, 0.1, 0, 0, 1.0)
    for i in range(B):
        n = int(lens[i]) * mul
        single = run_conv(lib, x[i:i + 1, :n].contiguous(), w, b, None, None, K, dil, None, 1, _abi.ACT_LRELU, 0.1, 0, 0, 1.0)
        assert torch.equal(out[i, :n], single[0])
        assert torch.count_nonzero(out[i, n:]) == 0
        ref = F.conv1d(F.leaky_relu(x[i:i + 1, :n].cpu().transpose(1, 2), 0.1), w.cpu().permute(2, 1, 0), b.cpu(),
                       padding=(K - 1) // 2 * dil, dilation=dil).transpose(1, 2)
        assert rel_max(single.cpu(), ref) <= TOL


def test_conv1d_per_item_bias(lib, dev):
    g = torch.Generator().manual_seed(12)
    B, L, Cin, Cout = 3, 40, 384, 384
    x = torch.randn(B, L, Cin, generator=g)
    w = torch.randn(Cin, Cout, generator=g) / math.sqrt(Cin)
    bias = torch.randn(B, Cout, generator=g)
    ref = x @ w + bias[:, None, :]
    out = run_conv(lib, x.to(dev), w.unsqueeze(0).contiguous().to(dev), bias.to(dev), None, None, 1, 1, None, 1, 0, 0.0, 0, 0, 1.0,
                   bias_bs=Cout)
    assert rel_max(out.cpu(), ref) <= TOL


@pytest.mark.parametrize("u,k,cin,cout", [(8, 16, 512, 256), (8, 16, 256, 128), (2, 4, 128, 64), (2, 4, 64, 32)])
def test_polyphase_transposed_conv(lib, dev, u, k, cin, cout):
    """ConvTranspose1d (hifigan/models.py:100-103) through the polyphase packing."""
    g = torch.Generator().manual_seed(u * 100 + cin)
    B, L = 2, 45
    x = torch.randn(B, cin, L, generator=g)
    w = torch.randn(cin, cout, k, generator=g) / math.sqrt(cin * 2)
    b = torch.randn(cout, generator=g)
    ref = F.conv_transpose1d(F.leaky_relu(x, 0.1), w, b, stride=u, padding=(k - u) // 2).transpose(1, 2)
    wp, bp = packing.polyphase_pack(w, b, u, (k - u) // 2)
    out = run_conv(lib, x.transpose(1, 2).contiguous().to(dev), wp.to(dev), bp.to(dev), None, None, wp.shape[0], 1, None, 1,
                   _abi.ACT_LRELU, 0.1, 0, 0, 1.0)
    assert rel_max(out.cpu().reshape(B, L * u, cout), ref) <= TOL


@pytest.mark.parametrize("tc_mode,tol", [(1, 2e-5), (0, 3e-3)], ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("B,L,masked", [(1, 7, False), (1, 64, False), (1, 129, False), (2, 500, True), (3, 1300, True), (1, 2049, False), (4, 65, True)])
def test_attention_tc(lib, dev, B, L, masked, tc_mode, tol):
    """encoder.py:84-109 on the tensor cores (csrc/attention_tc.cu): QK^T / PV as wgmma, softmax on the register accumulators.
    3xTF32 is held to the fp32 FFMA kernel's tolerance class (2e-5 of max|ref|); one tf32 MMA per step to 3e-3."""
    H, heads, dk = 384, 8, 48
    g = torch.Generator().manual_seed(L + 17 * B)
    qkv = torch.randn(B, L, 3 * H, generator=g)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32) if masked else None
    if masked:
        lens[0] = L
    q, k, v = [t.reshape(B, L, heads, dk).transpose(1, 2) for t in qkv.split(H, dim=-1)]
    scores = q @ k.transpose(-2, -1) / math.sqrt(dk)
    if masked:
        m = (torch.arange(L)[None, :] >= lens[:, None])[:, None, None, :]
        scores = scores.masked_fill(m, torch.finfo(torch.float32).min)
        attn = torch.softmax(scores, -1).masked_fill(m, 0.0)
    else:
        attn = torch.softmax(scores, -1)
    ref = (attn @ v).transpose(1, 2).reshape(B, L, H)
    out = torch.full((B, L, H), float("nan"), device=dev)
    qd = qkv.to(dev)
    ld = lens.to(dev) if masked else None
    _abi.check(lib.ev_op_attention_tc(qd.data_ptr(), _ptr(ld), out.data_ptr(), B, L, H, heads, tc_mode, _stream()))
    torch.cuda.synchronize()
    err = rel_max(out.cpu(), ref)
    print("attention_tc", (B, L, masked), tc_mode, "rel-max err %.2e" % err)
    assert err <= tol
    # batch invariance: item 1 of a masked batch is bitwise its own B=1 call on its valid prefix
    if masked and B > 1:
        n = int(lens[1])
        one = torch.empty(1, n, H, device=dev)
        q1 = qkv[1:2, :n].contiguous().to(dev)
        _abi.check(lib.ev_op_attention_tc(q1.data_ptr(), None, one.data_ptr(), 1, n, H, heads, tc_mode, _stream()))
        torch.cuda.synchronize()
        assert torch.equal(one[0], out[1, :n])


@pytest.mark.parametrize("tc_mode,tol", [(1, 2e-5), (0, 2e-2)], ids=["3xtf32", "tf32"])      # tf32: scores up to ~100 carry 2^-11 * 100 ~ 0.05
def test_attention_tc_lazy_rescale_path(lib, dev, tc_mode, tol):                               # in the exponent (inherent to tf32 operands)
    """The online softmax only rescales O / l when a key tile's row maximum exceeds the running one by more than 8.  Random
    scores never do, so this case makes them: the keys grow by a factor per 64-key tile (every tile after the first triggers
    the multiply of the accumulator registers), for some rows only (the warp-collective decision must leave the
    other rows exact), with a ragged second item."""
    H, heads, dk, B, L = 384, 8, 48, 2, 400
    g = torch.Generator().manual_seed(77)
    qkv = torch.randn(B, L, 3 * H, generator=g)
    scale = (1.0 + 2.5 * (torch.arange(L) // 64).float())[None, :, None]            # keys of later tiles are larger
    qkv[:, :, H:2 * H] *= scale
    qkv[:, 1::3, :H] *= 0.05                                                          # a third of the queries barely see it
    lens = torch.tensor([L, 333], dtype=torch.int32)
    q, k, v = [t.reshape(B, L, heads, dk).transpose(1, 2) for t in qkv.split(H, dim=-1)]
    scores = q.double() @ k.double().transpose(-2, -1) / math.sqrt(dk)
    m = (torch.arange(L)[None, :] >= lens[:, None])[:, None, None, :]
    attn = torch.softmax(scores.masked_fill(m, float("-inf")), -1)
    ref = (attn @ v.double()).transpose(1, 2).reshape(B, L, H).float()
    assert (scores.amax(-1) > 60).any()                                               # the jumps really exceed the threshold
    out = torch.full((B, L, H), float("nan"), device=dev)
    qd, ld = qkv.to(dev), lens.to(dev)
    _abi.check(lib.ev_op_attention_tc(qd.data_ptr(), ld.data_ptr(), out.data_ptr(), B, L, H, heads, tc_mode, _stream()))
    torch.cuda.synchronize()
    err = rel_max(out.cpu(), ref)
    print("attention_tc rescale path", tc_mode, "rel-max err %.2e" % err)
    assert err <= tol


@pytest.mark.parametrize("invariant", [0, 1])
def test_gauss_upsample(lib, dev, invariant):
    """alignment.py:180-211 incl. the cumsum; literal padded batch vs per-item semantics."""
    g = torch.Generator().manual_seed(3 + invariant)
    B, T, H = 3, 41, 384
    lens = torch.tensor([41, 9, 30], dtype=torch.int32)
    dur = torch.randint(0, 9, (B, T), generator=g)
    dur = dur * (torch.arange(T)[None, :] < lens[:, None])
    hs = torch.randn(B, T, H, generator=g)
    alpha = torch.tensor([1.3])
    dmask = torch.arange(T)[None, :] < lens[:, None]
    F_ = int(dur.sum(1).max())
    pe = packing.build_pe_table(F_, H)
    if invariant:
        ref = torch.zeros(B, F_, H)
        for b in range(B):
            n = int(lens[b])
            r, ml = O.gaussian_upsampling(hs[b:b + 1, :n], dur[b:b + 1, :n].clone(), dmask[b:b + 1, :n])
            ref[b, :r.shape[1]] = r[0] + alpha * pe[:r.shape[1]]
    else:
        ref, ml = O.gaussian_upsampling(hs, dur.clone(), dmask)
        ref = ref + alpha * pe[None]
    out = torch.empty(B, F_, H, device=dev)
    tmp = torch.empty(2 * B * T, device=dev)
    mel_lens = torch.empty(B + 1, dtype=torch.int32, device=dev)
    hd, dd, ld, pd, ad = hs.to(dev), dur.to(dev), lens.to(dev), pe.to(dev), alpha.to(dev)
    _abi.check(lib.ev_op_gauss_upsample(hd.data_ptr(), dd.data_ptr(), ld.data_ptr(), B, T, H, F_,
                                        invariant, pd.data_ptr(), ad.data_ptr(), tmp.data_ptr(),
                                        mel_lens.data_ptr(), out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    assert mel_lens.cpu().tolist() == dur.sum(1).tolist() + [F_]
    assert rel_max(out.cpu(), ref) <= TOL


def test_gauss_upsample_all_zero_durations(lib, dev):
    """alignment.py:187-191: if every duration is zero, every token gets duration 1."""
    B, T, H = 2, 5, 128
    lens = torch.tensor([5, 3], dtype=torch.int32)
    dur = torch.zeros(B, T, dtype=torch.int64)
    hs = torch.randn(B, T, H, generator=torch.Generator().manual_seed(1))
    dmask = torch.arange(T)[None, :] < lens[:, None]
    ref, ml = O.gaussian_upsampling(hs, dur.clone(), dmask)   # literal: F = T for all rows
    out = torch.empty(B, T, H, device=dev)
    tmp = torch.empty(2 * B * T, device=dev)
    mel_lens = torch.empty(B + 1, dtype=torch.int32, device=dev)
    hd, dd, ld = hs.to(dev), dur.to(dev), lens.to(dev)
    _abi.check(lib.ev_op_gauss_upsample(hd.data_ptr(), dd.data_ptr(), ld.data_ptr(), B, T, H, T, 0,
                                        None, None, tmp.data_ptr(), mel_lens.data_ptr(), out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    assert mel_lens.cpu().tolist() == [T, T, T]
    assert rel_max(out.cpu(), ref) <= TOL


def test_bad_arguments_return_error_codes(lib, dev):
    x = torch.zeros(1, 8, 30, device=dev)
    rc = lib.ev_op_conv1d(x.data_ptr(), x.data_ptr(), None, 0, None, x.data_ptr(), 1, 8, 30, 32, 3, 1, None, 1, 0, 0.0, 0, 0, 1.0, _stream())
    assert rc == -1 and b"Cin" in lib.ev_last_error()
    rc = lib.ev_op_conv1d(x.data_ptr(), x.data_ptr(), None, 0, None, x.data_ptr(), 1, 8, 32, 32, 4, 1, None, 1, 0, 0.0, 0, 0, 1.0, _stream())
    assert rc == -1 and b"odd" in lib.ev_last_error()
