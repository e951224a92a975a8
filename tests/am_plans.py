"""Host-side plans of the acoustic model's tensor-core convolutions and the list of launches ev_am_phase1 / ev_am_phase2 issue.

The plan function (ev_debug_tc_plan) runs without a device.  `engine_launches` restates the launch rules of csrc/engine.cu for
the reference configuration:
  * ev_am_phase1: validate_inputs, the embedding LayerNorm, the encoder (run_stack), the conditioning (gather, gemv, cond.wx),
    mask_rows in the literal batch (invariant = 0), the pitch / energy / duration predictors (run_predictor), var_embed_add and
    the duration scan;
  * ev_am_phase2: the Gaussian upsampling, the decoder (run_stack) and to_mel;
  * layer_run's choice of the kernel MODE: the duration-critical prefix (encoder, cond.wx, predictors) always runs 3xTF32
    (MODE 1); the decoder and to_mel run bf16x3 (MODE 3) in "fp32", 1xTF32 (MODE 0) in "tf32" and bf16 (MODE 2) in "bf16";
  * every layer's K-split factor S (kEncSplits, kDecSplits, 8 for the predictors, 4 for cond.wx, 2 for to_mel), clamped to
    the layer's C_in blocks, with one splitk_reduce launch after the convolution whenever the clamped S is > 1;
  * attention_tc (tc_mode 1 where the layer runs fp32-accurate, 0 otherwise) for d_k = 48, the FFMA attention for other
    head sizes.
  * in "fp32_ffma" every convolution runs the fp32 FFMA kernel (conv1d_tm, MODE FFMA here; no K split, so no reduce launch) and
    every attention the FFMA flash kernel.
A GPU test holds the length of this list to ev_launch_count(), so it cannot drift from engine.cu unnoticed.

The plan key of a convolution is (MODE, MT, KBG, BN, a_stages, b_stages, producer groups, ksplit): the template instantiation,
the tile width, and the ring depths and producer groups that fix the mbarrier protocol the kernel runs.  That of an FFMA
convolution is ("conv1d_tm", TXN, NV, TM): the template variant ev_debug_conv1d_plan reports.
"""
import ctypes

ACT_NONE, ACT_RELU, ACT_GELU = 0, 2, 3           # _abi.ACT_*
ENC_SPLITS = dict(qkv=4, wo=8, ffn1=4, ffn2=16)  # engine.cu kEncSplits
DEC_SPLITS = dict(qkv=2, wo=4, ffn1=4, ffn2=8)   # engine.cu kDecSplits
PRED_SPLIT, COND_SPLIT, MEL_SPLIT = 8, 4, 2
PREFIX_MODE = 1
FFMA = -1                                        # engine.cu kFfma: the fp32 FFMA kernel (conv1d_tm.cu) on the plain weights


def decoder_mode(prec):
    """Kernel MODE of the decoder's and to_mel's convolutions in a precision."""
    return {"fp32": 3, "tf32": 0, "bf16": 2, "fp32_ffma": FFMA}[prec]


def prefix_mode(prec):
    """Kernel MODE of the duration-critical prefix (encoder, cond.wx, predictors) in a precision."""
    return FFMA if prec == "fp32_ffma" else PREFIX_MODE


def conv1d_plan(lib, B, L, Cin, Cout, K, dil=1):
    """The plan ev_op_conv1d would use (ev_debug_conv1d_plan), or None for a shape it rejects."""
    v = (ctypes.c_int * 10)()
    if lib.ev_debug_conv1d_plan(B, L, Cin, Cout, K, dil, v) != 0:
        return None
    return dict(TXN=v[0], NV=v[1], TM=v[2], BM=v[3], BN=v[4], rows_a=v[5], a_ld=v[6], smem=v[7], grid=(v[8], v[9]),
                key=("conv1d_tm", v[0], v[1], v[2]))


def plan_of(lib, r):
    """Plan of one layer record of am_layers: the FFMA plan or the tensor-core one."""
    if r["mode"] == FFMA:
        return conv1d_plan(lib, r["B"], r["L"], r["Cin"], r["Cout"], r["K"])
    return tc_plan(lib, r["B"], r["L"], r["Cin"], r["Cout"], r["K"], r["mode"], r["ksplit"])


def tc_plan(lib, B, L, Cin, Cout, K, mode, ksplit):
    v = (ctypes.c_int * 11)()
    if lib.ev_debug_tc_plan(B, L, Cin, Cout, K, 1, mode, ksplit, v) != 0:
        return None
    return dict(BN=v[0], MT=v[1], KBG=v[2], a_stages=v[3], b_stages=v[4], groups=v[5], S=v[6], tiles=v[9],
                key=(mode, v[1], v[2], v[0], v[3], v[4], v[5], v[6]))


def am_shapes():
    from emotivoice_b200.config import default_config
    m = default_config().model
    return dict(H=int(m.encoder_n_hidden), heads=int(m.encoder_n_heads), enc=int(m.encoder_n_layers), dec=int(m.decoder_n_layers),
                ffn_k=int(m.encoder_kernel_size_conv_mod), pred_k=int(m.variance_kernel_size),
                preds=(("pitch", int(m.variance_n_layers)), ("energy", 2), ("dur", int(m.duration_n_layers))), n_mels=80)


def layer(name, B, L, Cin, Cout, K, mode, ksplit, bias_bs=0, inplace=False, out_act=ACT_NONE, lens=False):
    """One convolution launch of the engine: what the operator case must reproduce.  kind: the layer without its stack
    (enc.wo and dec.wo are both "wo"; the three predictors' convolutions are all "pred")."""
    kind = name.split(".", 1)[1] if name.startswith(("enc.", "dec.")) else ("pred" if name.endswith(".conv") else name)
    return dict(name=name, kind=kind, B=B, L=L, Cin=Cin, Cout=Cout, K=K, mode=mode, ksplit=ksplit, bias_bs=bias_bs, inplace=inplace,
                out_act=out_act, lens=lens)


def _stack(sh, tag, B, L, mode, splits, first_ln_done, conv_lens, attn_mode, out):
    H, K = sh["H"], sh["ffn_k"]
    n = sh["enc"] if tag == "enc" else sh["dec"]
    for i in range(n):
        if not (i == 0 and first_ln_done):
            out.append(("layernorm",))
        out.append(layer(tag + ".qkv", B, L, H, 3 * H, 1, mode, splits["qkv"], lens=conv_lens))
        out.append(("attention_tc", attn_mode) if H // sh["heads"] == 48 and mode != FFMA else ("attention",))
        out.append(layer(tag + ".wo", B, L, H, H, 1, mode, splits["wo"], inplace=True, lens=conv_lens))
        out.append(("layernorm",))
        out.append(layer(tag + ".ffn1", B, L, H, 4 * H, K, mode, splits["ffn1"], out_act=ACT_GELU, lens=conv_lens))
        out.append(layer(tag + ".ffn2", B, L, 4 * H, H, K, mode, splits["ffn2"], inplace=True, lens=conv_lens))
    out.append(("layernorm",))


def am_layers(B, T, F, prec, invariant, sh=None):
    """Every launch of one ev_am_phase1 + ev_am_phase2 call, in order: layer records (dicts) for the tensor-core convolutions,
    tuples for everything else.  The split-K reduce launches are not listed here (see engine_launches)."""
    sh = sh or am_shapes()
    H = sh["H"]
    inv = bool(invariant)
    pm = prefix_mode(prec)
    out = [("validate_inputs",), ("layernorm",)]
    _stack(sh, "enc", B, T, pm, ENC_SPLITS, True, inv, 1, out)
    out += [("cond_gather",), ("cond_gemv",),
            layer("cond.wx", B, T, H, H, 1, pm, COND_SPLIT, bias_bs=H, lens=inv)]
    if not inv:
        out.append(("mask_rows",))
    for name, n in sh["preds"]:
        for i in range(n):
            out.append(layer(name + ".conv", B, T, H, H, sh["pred_k"], pm, PRED_SPLIT, out_act=ACT_RELU, lens=inv))
            out.append(("layernorm",))
        out.append(("rowdot",))
    out += [("var_embed_add",), ("duration_scan",), ("gauss_upsample",)]
    dm = decoder_mode(prec)
    _stack(sh, "dec", B, F, dm, DEC_SPLITS, False, inv, 1 if dm in (1, 3) else 0, out)
    out.append(layer("to_mel", B, F, H, sh["n_mels"], 1, dm, MEL_SPLIT, lens=inv))
    return out


def engine_launches(lib, B, T, F, prec, invariant, sh=None):
    """Kernel launches of one Engine.acoustic call at (B, T phonemes, F frames): plan keys for the convolutions, each followed
    by ("splitk_reduce",) when its plan splits K, and the non-GEMM launches as tuples of their name."""
    out = []
    for r in am_layers(B, T, F, prec, invariant, sh):
        if isinstance(r, dict):
            p = plan_of(lib, r)
            assert p is not None, r
            out.append(p["key"])
            if r["mode"] != FFMA and p["S"] > 1:
                out.append(("splitk_reduce",))
        else:
            out.append(r)
    return out


def engine_conv_keys(lib, B, T, F, prec, invariant, sh=None):
    """{(layer kind, plan key)} of the convolutions of one call."""
    keys = set()
    for r in am_layers(B, T, F, prec, invariant, sh):
        if isinstance(r, dict):
            keys.add((r["kind"], plan_of(lib, r)["key"]))
    return keys
