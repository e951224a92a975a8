"""Host-side weight packing: reference state dict -> one fp32 blob + name index.

Runs once per ``load_state_dict`` (CPU torch ops: this is load-time plumbing, not the
compute path).  What it does, and the reference code each step replaces:

* nn.Linear (out,in) / nn.Conv1d (out,in,k) weights are re-laid to the engine's
  implicit-GEMM layout ``(k, C_in, C_out)`` (C_out contiguous).
* q/k/v projections of each attention block (encoder.py:72-82) are concatenated into
  one (H, 3H) matrix -> a single fused GEMM.
* ``embed_projection1`` (model_open_source.py:98,110-111) is split column-wise into the
  token part W_x (H,H) and the per-utterance part W_c (H+2*bert, H).
* weight-norm ``w = g * v / ||v||`` (hifigan/models.py:10-13, recomputed by the
  reference on EVERY forward for all 78 vocoder convs) is folded once.
* ConvTranspose1d (stride u, kernel k, padding p; hifigan/models.py:100-103) becomes a
  polyphase stride-1 convolution: output viewed as (L_in, u*C_out), phase r of the
  output reads input offsets ``q - i`` with weights ``W[:, :, j0 + i*u]`` where
  ``q, j0 = divmod(r + p, u)``.
"""
import ctypes
import math

import torch

from .synth import vocoder_conv_shapes


def build_pe_table(length, d_model):
    """Sinusoidal table of the reference's PositionalEncoding (encoder.py:223-237),
    evaluated with the same fp32 torch CPU ops so it is bit-identical."""
    pe = torch.zeros(length, d_model)
    position = torch.arange(0, length, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def _conv_w(w):          # (Cout, Cin, K) -> (K, Cin, Cout)
    return w.permute(2, 1, 0).contiguous()


def _lin_w(w):           # (out, in) -> (1, in, out)
    return w.t().contiguous().unsqueeze(0)


def round_tf32(w):
    """Round fp32 to the nearest tf32 (10 explicit mantissa bits, ties away from zero like
    cvt.rna.tf32.f32) so the tensor core's operand truncation is exact."""
    bits = w.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


TC_BN = 128     # widest N tile of the tensor-core kernel (csrc/conv1d_tc.cu); weights are blocked by it


def to_tc_layout(w_kio):
    """(K, Cin, Cout) -> (2, Cout/BNp, K, Cin/4, BNp, 4) with BNp = min(Cout, 128): the tensor-core
    kernel's weight layout.  Blocked by N tile, then granule-major: 16-byte K-granules with the tile's
    C_out rows 16 B apart, so one pipeline stage (tap, channel block) of one N tile is ONE contiguous run
    that a single bulk copy lands in shared memory exactly in the no-swizzle K-major wgmma operand layout.
    Plane 0 = tf32(w) ("hi"), plane 1 = tf32(w - hi) ("lo", used by the 3xTF32 fp32-emulation mode only)."""
    if w_kio.dim() == 2:
        w_kio = w_kio.unsqueeze(0)
    K, cin, cout = w_kio.shape
    assert cin % 4 == 0
    bnp = min(cout, TC_BN)
    assert cout % bnp == 0, "C_out must be <= 128 or a multiple of 128"
    g = w_kio.reshape(K, cin // 4, 4, cout // bnp, bnp).permute(3, 0, 1, 4, 2).contiguous()   # (NT, K, Cin/4, BNp, 4)
    hi = round_tf32(g)
    lo = round_tf32(g - hi)
    return torch.stack([hi, lo]).contiguous()


def to_tc16_layout(w_kio):
    """(K, Cin, Cout) -> bf16 (Cout/BNp, K, Cin/8, BNp, 8) viewed as fp32 words (..., 4): the bf16 variant of the
    tensor-core weight layout (8 channels per 16-byte granule, round to nearest even)."""
    if w_kio.dim() == 2:
        w_kio = w_kio.unsqueeze(0)
    K, cin, cout = w_kio.shape
    assert cin % 16 == 0, "bf16 tensor-core path needs C_in % 16 == 0"
    bnp = min(cout, TC_BN)
    assert cout % bnp == 0
    g = w_kio.reshape(K, cin // 8, 8, cout // bnp, bnp).permute(3, 0, 1, 4, 2).contiguous()   # (NT, K, Cin/8, BNp, 8)
    return g.to(torch.bfloat16).view(torch.float32)


def to_tc16x2_layout(w_kio):
    """(K, Cin, Cout) -> two bf16 planes in the tc16 layout, stacked: plane 0 = bf16(w) ("hi"), plane 1 = bf16(w - hi) ("lo").
    The "bf16x3" fp32 emulation of the vocoder (csrc/conv1d_gp.cu MODE 3): w ~= hi + lo to 16 significant bits."""
    if w_kio.dim() == 2:
        w_kio = w_kio.unsqueeze(0)
    hi = w_kio.to(torch.bfloat16)
    lo = (w_kio - hi.float()).to(torch.bfloat16)
    return torch.stack([to_tc16_layout(hi.float()), to_tc16_layout(lo.float())]).contiguous()


TC_SUFFIXES = ("wqkv", "wo", "w1", "w2")


def add_tc_weights(packed):
    """Adds '<name>.tc' copies for every GEMM-shaped layer that runs on the tensor cores: encoder and
    decoder stacks, conditioning W_x, predictor convs, to_mel and all vocoder convs but conv_post."""
    extra = {}
    for k, v in packed.items():
        last = k.rsplit(".", 1)[-1]
        is_stack = (k.startswith("enc.") or k.startswith("dec.")) and last in TC_SUFFIXES
        is_pred = k.split(".")[0] in ("dur", "pitch", "energy") and k.endswith(".w") and ".lin." not in k and ".ln." not in k
        is_voc = k.startswith("voc.") and k.endswith(".w") and k != "voc.post.w"
        if is_stack or is_pred or is_voc or k in ("to_mel.w", "cond.wx"):
            extra[k + ".tc"] = to_tc_layout(v)
        if (is_stack and k.startswith("dec.")) or is_voc or k == "to_mel.w":      # layers the bf16 mode runs in bf16
            extra[k + ".tc16"] = to_tc16_layout(v)
        if is_voc or (is_stack and k.startswith("dec.")) or k == "to_mel.w":     # the fp32 mode past the duration prefix: bf16x3 emulation
            extra[k + ".tc16x2"] = to_tc16x2_layout(v)
    packed.update(extra)
    return packed


def fold_weight_norm(sd, prefix):
    """Folded weight of a weight-normed conv, from either key convention
    (parametrizations.weight.original0/1, legacy weight_g/weight_v, or plain weight)."""
    for gk, vk in ((".parametrizations.weight.original0", ".parametrizations.weight.original1"),
                   (".weight_g", ".weight_v")):
        if prefix + gk in sd:
            return torch._weight_norm(sd[prefix + vk].float(), sd[prefix + gk].float(), 0)
    return sd[prefix + ".weight"].float()


def polyphase_pack(w, bias, stride, padding):
    """ConvTranspose1d weight (Cin, Cout, k) -> (K', Cin, stride*Cout) symmetric odd-K'
    stride-1 conv weight + tiled bias (stride*Cout).  See module docstring."""
    cin, cout, k = w.shape
    u, p = stride, padding
    taps = []
    for r in range(u):
        q, j0 = divmod(r + p, u)
        i = 0
        while j0 + i * u < k:
            taps.append((r, q - i, j0 + i * u))
            i += 1
    R = max(abs(o) for _, o, _ in taps)
    wp = torch.zeros(2 * R + 1, cin, u * cout, dtype=w.dtype)
    for r, o, j in taps:
        wp[o + R, :, r * cout:(r + 1) * cout] = w[:, :, j]
    return wp.contiguous(), bias.repeat(u).contiguous()


def pack_state_dict(sd, conf, prefix=""):
    """-> ordered dict name -> fp32 CPU tensor in the engine's layout.  ``sd`` uses the
    reference's JETSGenerator names (``am.*`` / ``generator.*``), optionally prefixed."""
    out = pack_state_dict_am(sd, conf, prefix)
    out.update(pack_vocoder(sd, conf.model, prefix + "generator."))
    return out


def pack_state_dict_am(sd, conf, prefix=""):
    """Acoustic-model part (``am.*`` keys; model_open_source.py:15-100)."""
    m = conf.model
    g = lambda k: sd[prefix + k].detach().float().cpu()
    out = {}
    out["emb.word"] = g("am.src_word_emb.weight")
    out["emb.spk"] = g("am.spk_tokenizer.weight")
    for name, ref, nl in (("enc", "am.encoder", m.encoder_n_layers), ("dec", "am.decoder", m.decoder_n_layers)):
        out[name + ".alpha"] = g(ref + ".embed.0.alpha").reshape(1)
        for i in range(nl):
            r = "%s.encoders.%d" % (ref, i)
            o = "%s.%d" % (name, i)
            out[o + ".ln1.w"], out[o + ".ln1.b"] = g(r + ".norm1.weight"), g(r + ".norm1.bias")
            out[o + ".wqkv"] = torch.cat([g(r + ".self_attn.linear_%s.weight" % n).t() for n in "qkv"], dim=1).contiguous()
            out[o + ".bqkv"] = torch.cat([g(r + ".self_attn.linear_%s.bias" % n) for n in "qkv"])
            out[o + ".wo"], out[o + ".bo"] = _lin_w(g(r + ".self_attn.linear_out.weight")), g(r + ".self_attn.linear_out.bias")
            out[o + ".ln2.w"], out[o + ".ln2.b"] = g(r + ".norm2.weight"), g(r + ".norm2.bias")
            out[o + ".w1"], out[o + ".b1"] = _conv_w(g(r + ".feed_forward.w_1.weight")), g(r + ".feed_forward.w_1.bias")
            out[o + ".w2"], out[o + ".b2"] = _conv_w(g(r + ".feed_forward.w_2.weight")), g(r + ".feed_forward.w_2.bias")
        out[name + ".lnf.w"], out[name + ".lnf.b"] = g(ref + ".after_norm.weight"), g(ref + ".after_norm.bias")
    H = m.encoder_n_hidden
    W = g("am.embed_projection1.weight")           # (H, 2H + 2*bert): [x | spk | style | content]
    out["cond.wx"] = W[:, :H].t().contiguous()
    out["cond.wc"] = W[:, H:].t().contiguous()
    out["cond.b"] = g("am.embed_projection1.bias")
    for name, ref, nl in (("dur", "am.duration_predictor", m.duration_n_layers),
                          ("pitch", "am.pitch_predictor", m.variance_n_layers),
                          ("energy", "am.energy_predictor", 2)):
        for i in range(nl):
            out["%s.%d.w" % (name, i)] = _conv_w(g("%s.conv.%d.0.weight" % (ref, i)))
            out["%s.%d.b" % (name, i)] = g("%s.conv.%d.0.bias" % (ref, i))
            out["%s.%d.ln.w" % (name, i)] = g("%s.conv.%d.2.weight" % (ref, i))
            out["%s.%d.ln.b" % (name, i)] = g("%s.conv.%d.2.bias" % (ref, i))
        out[name + ".lin.w"] = g(ref + ".linear.weight").reshape(-1)
        out[name + ".lin.b"] = g(ref + ".linear.bias").reshape(1)
    out["pitch_emb.w"] = g("am.pitch_embed.0.weight")[:, 0, :].t().contiguous()     # (K, H)
    out["pitch_emb.b"] = g("am.pitch_embed.0.bias")
    out["energy_emb.w"] = g("am.energy_embed.0.weight")[:, 0, :].t().contiguous()
    out["energy_emb.b"] = g("am.energy_embed.0.bias")
    out["to_mel.w"], out["to_mel.b"] = _lin_w(g("am.to_mel.weight")), g("am.to_mel.bias")
    return out


def pack_vocoder(sd, h, prefix="generator."):
    """Folded + re-laid HiFi-GAN generator weights (hifigan/models.py:90-113)."""
    sdc = {k: v.detach().float().cpu() for k, v in sd.items() if k.startswith(prefix)}
    out = {}
    nk = len(h.resblock_kernel_sizes)
    for mod, shape, transposed in vocoder_conv_shapes(h):
        w = fold_weight_norm(sdc, prefix + mod)
        b = sdc[prefix + mod + ".bias"]
        if mod == "conv_pre":
            out["voc.pre.w"], out["voc.pre.b"] = _conv_w(w), b
        elif mod == "conv_post":
            out["voc.post.w"], out["voc.post.b"] = w[0].t().contiguous(), b.reshape(1)      # (K, C)
        elif transposed:
            i = int(mod.split(".")[1])
            u, k = h.upsample_rates[i], h.upsample_kernel_sizes[i]
            out["voc.up.%d.w" % i], out["voc.up.%d.b" % i] = polyphase_pack(w, b, u, (k - u) // 2)
        else:
            _, n, grp, l = mod.split(".")
            c = "c1" if grp == "convs1" else "c2"
            out["voc.rb.%s.%s.%s.w" % (n, c, l)], out["voc.rb.%s.%s.%s.b" % (n, c, l)] = _conv_w(w), b
    return out


class WeightEntry(ctypes.Structure):
    """ev_weight_entry (include/emotivoice_b200.h)."""
    _fields_ = [("name", ctypes.c_char * 56), ("offset", ctypes.c_uint64), ("numel", ctypes.c_uint64)]


def make_blob(packed, align=64):
    """Concatenate into one contiguous fp32 CPU tensor (each tensor 256-byte aligned)
    and build the ctypes index."""
    offs, total = {}, 0
    for k, v in packed.items():
        offs[k] = total
        total += (v.numel() + align - 1) // align * align
    blob = torch.zeros(total, dtype=torch.float32)
    index = (WeightEntry * len(packed))()
    for i, (k, v) in enumerate(packed.items()):
        assert len(k) < 56, k
        blob[offs[k]:offs[k] + v.numel()] = v.reshape(-1)
        index[i].name = k.encode()
        index[i].offset = offs[k]
        index[i].numel = v.numel()
    return blob, index


def index_from_meta(meta):
    """[(name, offset, numel)] -> the ctypes index ``make_blob`` builds (for a blob received from another rank)."""
    index = (WeightEntry * len(meta))()
    for i, (k, off, n) in enumerate(meta):
        index[i].name = k.encode()
        index[i].offset = int(off)
        index[i].numel = int(n)
    return index


# ---- style encoder (simbert.py:33-72; transformers BertModel names under ``bert.``) ---------------------------------

STYLE_HEADS = ("pitch", "speed", "energy", "emotion")      # order of the packed classifier columns (simbert.py:58-61)


def style_head_slices(sc):
    """name -> (first column, n_labels) inside the packed ``sty.heads`` output; total padded to a multiple of 8."""
    out, c = {}, 0
    for n in STYLE_HEADS:
        k = int(getattr(sc, n + "_n_labels"))
        out[n] = (c, k)
        c += k
    return out, (c + 7) // 8 * 8


def pack_style_state_dict(sd, sc, prefix=""):
    """Reference StyleEncoder state dict -> engine layout ("sty.*").  Linear weights go straight to the tensor-core layout
    (two tf32 planes; no plain fp32 copy: the style encoder has no FFMA mode), q|k|v are fused into one (H, 3H) GEMM, the
    pooler / classifier matrices are stored (K, N) row-major for the GEMV kernel, the four heads side by side."""
    g = lambda k: sd[prefix + k].detach().float().cpu()
    H = sc.hidden_size
    out = {}
    e = "bert.embeddings."
    out["sty.emb.word"], out["sty.emb.pos"] = g(e + "word_embeddings.weight"), g(e + "position_embeddings.weight")
    out["sty.emb.type"] = g(e + "token_type_embeddings.weight")
    out["sty.emb.ln.w"], out["sty.emb.ln.b"] = g(e + "LayerNorm.weight"), g(e + "LayerNorm.bias")
    for i in range(sc.num_hidden_layers):
        r, o = "bert.encoder.layer.%d." % i, "sty.%d" % i
        wqkv = torch.cat([g(r + "attention.self.%s.weight" % n).t() for n in ("query", "key", "value")], dim=1).contiguous()
        out[o + ".wqkv.tc"] = to_tc_layout(wqkv.unsqueeze(0))
        out[o + ".bqkv"] = torch.cat([g(r + "attention.self.%s.bias" % n) for n in ("query", "key", "value")])
        out[o + ".wo.tc"], out[o + ".bo"] = to_tc_layout(_lin_w(g(r + "attention.output.dense.weight"))), g(r + "attention.output.dense.bias")
        out[o + ".ln1.w"], out[o + ".ln1.b"] = g(r + "attention.output.LayerNorm.weight"), g(r + "attention.output.LayerNorm.bias")
        out[o + ".w1.tc"], out[o + ".b1"] = to_tc_layout(_lin_w(g(r + "intermediate.dense.weight"))), g(r + "intermediate.dense.bias")
        out[o + ".w2.tc"], out[o + ".b2"] = to_tc_layout(_lin_w(g(r + "output.dense.weight"))), g(r + "output.dense.bias")
        out[o + ".ln2.w"], out[o + ".ln2.b"] = g(r + "output.LayerNorm.weight"), g(r + "output.LayerNorm.bias")
    out["sty.pool.w"], out["sty.pool.b"] = g("bert.pooler.dense.weight").t().contiguous(), g("bert.pooler.dense.bias")
    slices, width = style_head_slices(sc)
    hw, hb = torch.zeros(H, width), torch.zeros(width)
    for n, (c0, k) in slices.items():
        hw[:, c0:c0 + k] = g(n + "_clf.classifier.weight").t()
        hb[c0:c0 + k] = g(n + "_clf.classifier.bias")
    out["sty.heads.w"], out["sty.heads.b"] = hw.contiguous(), hb
    return out
