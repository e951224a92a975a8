"""Tensor-core implicit-GEMM convolution (conv1d_tc.cu) and the precision modes of the engine.

Per-operator tolerances against a torch fp32 CPU reference:
  1xTF32 (operands rounded to nearest tf32, 10-bit mantissa, fp32 accumulation): 3e-3 * max|ref|
  3xTF32 (fp32 emulation: hi/lo split, three MMAs per K step):                          5e-5 * max|ref|
    (measured 2e-6 .. 2.1e-5, the largest at K = 3*1536; the fp32 FFMA kernel is held to 2e-5).
End to end in "tf32" mode: mel <= 5e-3 * max|mel|, wav rms <= 2e-2 * rms(wav); durations identical in
every mode (the duration-critical prefix is always fp32-accurate)."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden, rel_max, rel_rms
from emotivoice_b200 import _abi, packing

pytestmark = pytest.mark.gpu
TOL = {0: 3e-3, 1: 5e-5, 2: 1.5e-2}      # mode -> tolerance (3xTF32: K up to 4608-term fp32 sums, measured <= 2.1e-5;
                                        # bf16: 8-bit mantissa operands, rel 2^-9 each)
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")


def _ptr(t):
    return None if t is None else t.data_ptr()


def run_tc(lib, split3, x_tm, w_kio, bias, res, out_init, K, dil, lens, lens_mul, in_act, in_slope, out_act, acc, div, bias_bs=0, ws=None):
    B, L, Cin = x_tm.shape
    Cout = w_kio.shape[2]
    w_tc = (packing.to_tc16_layout(w_kio.cpu()) if split3 == 2 else packing.to_tc_layout(w_kio.cpu())).to(x_tm.device)
    out = out_init.clone() if out_init is not None else torch.full((B, L, Cout), float("nan"), device=x_tm.device)
    _abi.check(lib.ev_op_conv1d_tc(_ptr(x_tm), _ptr(w_tc), split3, _ptr(bias), bias_bs, _ptr(res), _ptr(out), B, L, Cin, Cout, K, dil,
                                   _ptr(lens), lens_mul, in_act, in_slope, out_act, acc, div, _ptr(ws), 0 if ws is None else ws.numel(),
                                   torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out


TC_CASES = [
    # B, L, Cin, Cout, K, dil
    (1, 128, 32, 32, 1, 1),       # one tile, one K block, one tap
    (1, 128, 64, 32, 1, 1),       # two K blocks
    (1, 128, 32, 32, 3, 1),       # taps: row-shifted descriptor start addresses
    (1, 300, 32, 32, 11, 5),      # widest receptive field, ragged last tile
    (2, 517, 64, 64, 7, 3),
    (1, 100, 384, 1152, 1, 1),    # fused q|k|v projection: 9 N tiles
    (1, 260, 384, 1536, 3, 1),    # conv-FFN 1
    (2, 130, 1536, 384, 3, 1),    # conv-FFN 2 (48 K blocks)
    (1, 70, 80, 512, 7, 1),       # conv_pre: C_in tail block of 16
    (3, 700, 128, 128, 3, 1),
    (2, 900, 256, 256, 11, 1),    # N = 256 single tile
    (1, 537, 384, 80, 1, 1),      # to_mel: N = 80
    (1, 5000, 32, 32, 3, 3),
    (3, 70000, 32, 32, 11, 5),    # persistent: many tiles per CTA, N = 32 (half of the epilogue warps idle)
    (2, 40000, 64, 64, 3, 1),     # persistent, MT = 4
]


def check_conv1d_tc_matches_torch(lib, dev, B, L, Cin, Cout, K, dil, split3):
    g = torch.Generator().manual_seed(B * 1000 + L + Cin + Cout + K)
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g)
    ref = F.conv1d(F.leaky_relu(x, 0.1), w, b, padding=(K - 1) // 2 * dil, dilation=dil).transpose(1, 2)
    out = run_tc(lib, split3, x.transpose(1, 2).contiguous().to(dev), packing._conv_w(w), b.to(dev), None, None,
                 K, dil, None, 1, _abi.ACT_LRELU, 0.1, _abi.ACT_NONE, _abi.ACC_STORE, 1.0)
    err = rel_max(out.cpu(), ref)
    print("tc conv", (B, L, Cin, Cout, K, dil), ("1xTF32", "3xTF32", "bf16")[split3], "rel-max err %.2e" % err)
    assert err <= TOL[split3]


@pytest.mark.parametrize("split3", [0, 1])
@pytest.mark.parametrize("B,L,Cin,Cout,K,dil", TC_CASES)
def test_conv1d_tc_matches_torch(lib, dev, B, L, Cin, Cout, K, dil, split3):
    check_conv1d_tc_matches_torch(lib, dev, B, L, Cin, Cout, K, dil, split3)


def check_conv1d_tc_epilogue_and_ragged(lib, dev, split3):
    g = torch.Generator().manual_seed(21)
    B, L, C, K, dil, mul = 3, 96 * 4, 64, 7, 3, 4
    lens = torch.tensor([96, 17, 50], dtype=torch.int32)
    x = torch.randn(B, L, C, generator=g).to(dev)
    w = torch.randn(K, C, C, generator=g) / math.sqrt(C * K)
    b = torch.randn(C, generator=g).to(dev)
    res = torch.randn(B, L, C, generator=g).to(dev)
    prev = torch.randn(B, L, C, generator=g).to(dev)
    out = run_tc(lib, split3, x, w, b, res, prev, K, dil, lens.to(dev), mul, _abi.ACT_LRELU, 0.1, _abi.ACT_GELU, _abi.ACC_ADD_DIV, 3.0)
    for i in range(B):
        n = int(lens[i]) * mul
        y = F.conv1d(F.leaky_relu(x[i:i + 1, :n].cpu().transpose(1, 2), 0.1), w.permute(2, 1, 0), b.cpu(),
                     padding=(K - 1) // 2 * dil, dilation=dil).transpose(1, 2)
        ref = (prev[i:i + 1, :n].cpu() + (F.gelu(y) + res[i:i + 1, :n].cpu())) / 3.0
        assert rel_max(out[i:i + 1, :n].cpu(), ref) <= TOL[split3]
        assert torch.count_nonzero(out[i, n:]) == 0
        single = run_tc(lib, split3, x[i:i + 1, :n].contiguous(), w, b, res[i:i + 1, :n].contiguous(), prev[i:i + 1, :n].contiguous(),
                        K, dil, None, 1, _abi.ACT_LRELU, 0.1, _abi.ACT_GELU, _abi.ACC_ADD_DIV, 3.0)
        assert torch.equal(single[0], out[i, :n])           # batch-invariant, bitwise


@pytest.mark.parametrize("split3", [0, 1])
def test_conv1d_tc_epilogue_and_ragged(lib, dev, split3):
    check_conv1d_tc_epilogue_and_ragged(lib, dev, split3)


@pytest.mark.parametrize("split3", [0, 1])
def test_conv1d_tc_split_k_is_deterministic_and_matches(lib, dev, split3):
    """Few output tiles + long reduction (the conv-FFN's second conv): K-split over CTAs with private
    partial buffers and a fixed-order reduce.  Same tolerance; bitwise reproducible; epilogue fused in
    the reduce kernel (bias, GELU, residual, accumulate)."""
    g = torch.Generator().manual_seed(31)
    B, L, Cin, Cout, K = 1, 300, 1536, 384, 3
    x = torch.randn(B, L, Cin, generator=g).to(dev)
    w = torch.randn(K, Cin, Cout, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g).to(dev)
    res = torch.randn(B, L, Cout, generator=g).to(dev)
    prev = torch.randn(B, L, Cout, generator=g).to(dev)
    ws = torch.empty(8 * B * L * Cout, device=dev)
    y = F.conv1d(x.cpu().transpose(1, 2), w.permute(2, 1, 0), b.cpu(), padding=1).transpose(1, 2)
    ref = (prev.cpu() + (F.gelu(y) + res.cpu())) / 3.0
    o1 = run_tc(lib, split3, x, w, b, res, prev, K, 1, None, 1, 0, 0.0, _abi.ACT_GELU, _abi.ACC_ADD_DIV, 3.0, ws=ws)
    o2 = run_tc(lib, split3, x, w, b, res, prev, K, 1, None, 1, 0, 0.0, _abi.ACT_GELU, _abi.ACC_ADD_DIV, 3.0, ws=ws)
    o0 = run_tc(lib, split3, x, w, b, res, prev, K, 1, None, 1, 0, 0.0, _abi.ACT_GELU, _abi.ACC_ADD_DIV, 3.0, ws=None)
    assert torch.equal(o1, o2)
    assert rel_max(o1.cpu(), ref) <= TOL[split3] and rel_max(o0.cpu(), ref) <= TOL[split3]


@pytest.mark.parametrize("name", ["b1_t12", "b1_t100"])
def test_tf32_mode_end_to_end(model, dev, name):
    g = load_golden(name)
    model.precision = "tf32"
    try:
        out = model(**{k: g[k].to(dev) for k in KEYS})
        torch.cuda.synchronize()
    finally:
        model.precision = "fp32"
    assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
    e_mel, e_wav = rel_max(out["dec_outputs"].cpu(), g["mel"]), rel_rms(out["wav_predictions"].cpu(), g["wav"])
    print(name, "tf32: mel rel-max %.2e wav rms-rel %.2e" % (e_mel, e_wav))
    assert e_mel <= 5e-3 and e_wav <= 2e-2


def test_tf32_mode_is_batch_invariant(model, dev):
    from emotivoice_b200 import synth
    g = load_golden("b3_padded")
    model.precision = "tf32"
    try:
        out = model(**{k: g[k].to(dev) for k in KEYS})
        for b in range(3):
            single = model(**{k: v.to(dev) for k, v in synth.slice_batch(g, b).items()})
            Fb = single["dec_outputs"].shape[1]
            assert torch.equal(single["dec_outputs"][0], out["dec_outputs"][b, :Fb])
            assert torch.equal(single["wav_predictions"][0, 0], out["wav_predictions"][b, 0, :Fb * 256])
    finally:
        model.precision = "fp32"


@pytest.mark.parametrize("B,L,Cin,Cout,K", [(1, 537, 384, 1152, 1), (1, 537, 384, 1536, 3), (2, 130, 1536, 384, 3), (1, 537, 384, 80, 1), (3, 700, 128, 128, 3)])
def test_conv1d_tc_bf16x3_is_fp32_class(lib, dev, B, L, Cin, Cout, K):
    """MODE 3 of conv1d_tc ("bf16x3": fp32 operands split into bf16 hi + lo, three kind::f16 MMAs per K = 16 step) -- what the
    decoder's GEMM-shaped layers run in the "fp32" precision.  Against an fp64 torch reference: <= 5e-5 of max|ref|
    (16 significant bits per operand; 3xTF32 is held to the same bound), with the GELU / residual epilogue and K-split."""
    g = torch.Generator().manual_seed(B + L + Cin + Cout + K)
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g)
    res = torch.randn(B, L, Cout, generator=g)
    ref = F.gelu(F.conv1d(x.double(), w.double(), b.double(), padding=(K - 1) // 2)).transpose(1, 2) + res.double()
    xd, bd, rd = x.transpose(1, 2).contiguous().to(dev), b.to(dev), res.to(dev)
    wd = packing.to_tc16x2_layout(packing._conv_w(w)).to(dev)
    for ws_floats in (0, 4 * B * L * Cout):
        ws = torch.empty(ws_floats, device=dev) if ws_floats else None
        out = torch.full((B, L, Cout), float("nan"), device=dev)
        _abi.check(lib.ev_op_conv1d_tc(_ptr(xd), _ptr(wd), 3, _ptr(bd), 0, _ptr(rd), _ptr(out), B, L, Cin, Cout, K, 1, None, 1, _abi.ACT_NONE, 0.0,
                                       _abi.ACT_GELU, _abi.ACC_STORE, 1.0, _ptr(ws), ws_floats, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        err = float((out.cpu().double() - ref).abs().max() / ref.abs().max())
        print("conv1d_tc bf16x3", (B, L, Cin, Cout, K), "ksplit" if ws_floats else "plain", "rel-max err %.2e" % err)
        assert err <= 5e-5
