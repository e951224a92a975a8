"""Host-side list of the launches ev_style_forward issues, and the plans of its tensor-core GEMMs.

`style_launches` restates the launch rules of csrc/style_engine.cu (ev_style_forward) for a style configuration
(emotivoice_b200.synth.style_config: BERT-base, or the 2-layer "small" model):
  * validate_inputs, then bert_embed_ln;
  * per layer: qkv (H -> 3H, S = 2), attention (the FFMA kernel, launch_attention, for every head size), wo (H -> H, S = 2,
    residual x, out y), layernorm, ffn1 (H -> I, S = 2, GELU), ffn2 (I -> H, S = 4, residual x, out y), layernorm;
  * the pooler row_gemv, and the heads row_gemv when the call asks for them (n_head_out > 0);
  * the kernel MODE of every GEMM: 1 (3xTF32) in "fp32", 0 (1xTF32) in "tf32";
  * one splitk_reduce after each GEMM whose K-split factor, clamped to its C_in blocks, is > 1.
A GPU test holds the length of this list to ev_launch_count(), so it cannot drift from style_engine.cu unnoticed.

The plan key carries no C_in or C_out, so the layer kinds are kept apart per configuration: "base:sty.qkv", "small:sty.ffn2", ...
"""
import am_plans

ACT_NONE, ACT_GELU = am_plans.ACT_NONE, am_plans.ACT_GELU
SPLITS = {"qkv": 2, "wo": 2, "ffn1": 2, "ffn2": 4}      # style_engine.cu: the ksplit argument of each style_gemm
CONFIGS = ("base", "small")
KINDS = ("qkv", "wo", "ffn1", "ffn2")


def style_mode(prec):
    """Kernel MODE of the style GEMMs in a precision (style_gemm: EV_PREC_TF32 -> 0, else 1)."""
    return {"fp32": 1, "tf32": 0}[prec]


def style_config(cfg):
    from emotivoice_b200 import synth
    return synth.style_config(cfg == "small")


def kind_name(cfg, kind):
    return "%s:sty.%s" % (cfg, kind)


def layer_table(cfg):
    """kind -> (Cin, Cout, K, out_act, residual, per-item bias, input is a GELU output) of the configuration's four GEMMs, in
    the form of am_cases.KINDS.  The residual of wo and ffn2 is x, read from another buffer than the output y ("separate")."""
    sc = style_config(cfg)
    H, I = int(sc.hidden_size), int(sc.intermediate_size)
    return {kind_name(cfg, "qkv"): (H, 3 * H, 1, ACT_NONE, None, False, False),
            kind_name(cfg, "wo"): (H, H, 1, ACT_NONE, "separate", False, False),
            kind_name(cfg, "ffn1"): (H, I, 1, ACT_GELU, None, False, False),
            kind_name(cfg, "ffn2"): (I, H, 1, ACT_NONE, "separate", False, True)}


def _n_head_out(sc):
    from emotivoice_b200 import packing
    return packing.style_head_slices(sc)[1]


def style_layers(cfg, B, N, prec, heads=True):
    """Every launch of one ev_style_forward call at (B items, N tokens), in order: GEMM records (dicts) for the tensor-core
    convolutions, tuples for everything else.  The split-K reduce launches are not listed here (see style_launches)."""
    sc = style_config(cfg)
    tab = layer_table(cfg)
    mode = style_mode(prec)
    out = [("validate_inputs",), ("bert_embed_ln",)]

    def gemm(kind):
        Cin, Cout, K, act, res = tab[kind_name(cfg, kind)][:5]
        return dict(kind=kind_name(cfg, kind), B=B, L=N, Cin=Cin, Cout=Cout, K=K, mode=mode, ksplit=SPLITS[kind], out_act=act,
                    res=res)

    for _ in range(int(sc.num_hidden_layers)):
        out += [gemm("qkv"), ("attention",), gemm("wo"), ("layernorm",), gemm("ffn1"), gemm("ffn2"), ("layernorm",)]
    out.append(("row_gemv", "pooler"))
    if heads and _n_head_out(sc) > 0:
        out.append(("row_gemv", "heads"))
    return out


def style_launches(lib, cfg, B, N, prec, heads=True):
    """Kernel launches of one ev_style_forward call: plan keys for the GEMMs, each followed by ("splitk_reduce",) when its plan
    splits K, and the other launches as tuples of their name."""
    out = []
    for r in style_layers(cfg, B, N, prec, heads):
        if isinstance(r, dict):
            p = am_plans.tc_plan(lib, r["B"], r["L"], r["Cin"], r["Cout"], r["K"], r["mode"], r["ksplit"])
            assert p is not None, r
            out.append(p["key"])
            if p["S"] > 1:
                out.append(("splitk_reduce",))
        else:
            out.append(r)
    return out


def style_conv_keys(lib, cfg, B, N, prec):
    """{(layer kind, plan key)} of the GEMMs of one call (every layer of a kind launches the same plan)."""
    layers = {r["kind"]: r for r in style_layers(cfg, B, N, prec) if isinstance(r, dict)}
    return {(k, am_plans.tc_plan(lib, r["B"], r["L"], r["Cin"], r["Cout"], r["K"], r["mode"], r["ksplit"])["key"])
            for k, r in layers.items()}
