"""Host-side plans of the vocoder's granule-planar kernels and the list of launches ev_vocoder issues.

The plan functions (ev_debug_*plan) run without a device; sm_count() then assumes an H100's 132 SMs.  `engine_launches`
restates the launch rules of ev_vocoder (csrc/engine.cu) for the reference configuration:
  * grouped launches of the three parallel ResBlocks while B*F <= 2400 (the stage-buffer rule of carve_voc) and one member
    alone has fewer than two waves of tiles, with an elementwise pass forming xs / 3 after a grouped last layer (fp32 storage);
  * otherwise one launch per ResBlock layer, fused (resblock_gp) where the fused plan keeps at least two accumulators per tile
    and not for C >= 64 with k > 7 once B * L > 280 000; two conv1d_gp launches where it is not fused.
In "fp32_ffma" (MODE FFMA) the vocoder runs on time-major activations: a transpose for a channels-first mel only, then one
conv1d_tm launch per convolution (conv_pre, each polyphase up, c1 and c2 of every ResBlock layer, in engine order) and
conv_post.
A GPU test holds this list to ev_launch_count(), so it cannot drift from engine.cu unnoticed.
"""
import ctypes

import am_plans

NSM = 132
GROUP_MAX_FRAMES = 2400           # carve_voc / voc_group_frames
UNFUSE_BL = 4 * 70000             # try_gp_pair: C >= 64 and k > 7 run unfused above this many batch-rows

_IA = lambda v: (ctypes.c_int * len(v))(*v)


def gp_plan(lib, B, L, Cin, Cout, K, dil, rate, mode):
    v = (ctypes.c_int * 11)()
    if lib.ev_debug_gp_plan(B, L, Cin, Cout, K, dil, rate, mode, v) != 0:
        return None
    return dict(BN=v[0], MT=v[1], KBG=v[2], tiles=v[9], key=("conv1d_gp", mode, v[1], v[2], v[0], rate))


def gp_group_plan(lib, Ks, dils, B, L, Cin, Cout, mode):
    v = (ctypes.c_int * 11)()
    if lib.ev_debug_gp_group_plan(len(Ks), _IA(Ks), _IA(dils), B, L, Cin, Cout, mode, v) != 0:
        return None
    return dict(BN=v[0], MT=v[1], KBG=v[2], tiles=v[9], key=("conv1d_gp_group", mode, v[1], v[2], v[0], 1))


def pair_plan(lib, B, L, C, K, dil, mode):
    v = (ctypes.c_int * 11)()
    if lib.ev_debug_resblock_gp_plan(B, L, C, K, dil, mode, v) != 0:
        return None
    return dict(MT=v[0], KBG=v[1], tiles=v[7], R=v[8], key=("resblock_gp", mode, v[0], v[1], C, 1))


def pair_group_plan(lib, Ks, dils, B, L, C, mode):
    v = (ctypes.c_int * 16)()
    if lib.ev_debug_resblock_gp_group_plan(len(Ks), _IA(Ks), _IA(dils), B, L, C, mode, v) != 0:
        return None
    members = [dict(K=v[7 + 3 * i], tiles_m=v[8 + 3 * i], tile0=v[9 + 3 * i]) for i in range(len(Ks))]
    return dict(MT=v[0], KBG=v[1], tiles=v[2], members=members, key=("resblock_gp_group", mode, v[0], v[1], C, 1))


def voc_shapes():
    """The reference configuration's vocoder: conv_pre, the polyphase ups (Cin, packed Cout, taps, rate) and the ResBlocks."""
    import torch
    from emotivoice_b200 import packing
    from emotivoice_b200.config import default_config
    h = default_config().model
    c0 = int(h.upsample_initial_channel)
    ups = []
    for s, (u, k) in enumerate(zip(h.upsample_rates, h.upsample_kernel_sizes)):
        cin, cout = c0 // 2 ** s, c0 // 2 ** (s + 1)
        taps = packing.polyphase_pack(torch.zeros(1, 1, k), torch.zeros(1), u, (k - u) // 2)[0].shape[0]
        ups.append(dict(cin=cin, cout=cout, rate=int(u), K=taps))
    return dict(n_mels=80, c0=c0, pre_k=7, ups=ups, res_k=[int(k) for k in h.resblock_kernel_sizes],
                res_d=[[int(d) for d in ds] for ds in h.resblock_dilation_sizes])


def _fused(lib, B, L, C, K, dil, mode):
    if C >= 64 and K > 7 and B * L > UNFUSE_BL:
        return None
    p = pair_plan(lib, B, L, C, K, dil, mode)
    return p if p is not None and p["MT"] >= 2 else None


def _grouped_stage(lib, B, L, C, Ks, Ds, mode):
    J, D = len(Ks), len(Ds[0])
    if not 2 <= J <= 3:
        return None
    fused = [[_fused(lib, B, L, C, Ks[j], Ds[j][l], mode) for j in range(J)] for l in range(D)]
    n_pair = sum(p is not None for row in fused for p in row)
    out = []
    if n_pair == J * D:
        groups = [pair_group_plan(lib, Ks, [Ds[j][l] for j in range(J)], B, L, C, mode) for l in range(D)]
        if any(g is None for g in groups) or fused[D - 1][0]["tiles"] >= 2 * NSM:
            return None
        for l in range(D):
            last = l == D - 1
            sum_pass = last and mode != 2 and D >= 2
            if not last or sum_pass:
                out.append(groups[l]["key"])
                if sum_pass:
                    out.append(("gp_sum_div",))
            else:
                out += [fused[l][j]["key"] for j in range(J)]
        return out
    if n_pair:
        return None
    g1 = [gp_group_plan(lib, Ks, [Ds[j][l] for j in range(J)], B, L, C, C, mode) for l in range(D)]
    g2 = gp_group_plan(lib, Ks, [1] * J, B, L, C, C, mode)
    if any(g is None for g in g1) or g2 is None or gp_plan(lib, B, L, C, C, Ks[0], 1, 1, mode)["tiles"] >= 2 * NSM:
        return None
    for l in range(D):
        last = l == D - 1
        sum_pass = last and mode != 2 and D >= 2
        out.append(g1[l]["key"])
        if not last or sum_pass:
            out.append(g2["key"])
            if sum_pass:
                out.append(("gp_sum_div",))
        else:
            out += [gp_plan(lib, B, L, C, C, K, 1, 1, mode)["key"] for K in Ks]
    return out


def ffma_layers(B, F, shapes=None):
    """The convolutions ev_vocoder runs in "fp32_ffma" at (B, F), in order: dicts of the layer (kind: "pre", "ups<s>",
    "c1_C<C>", "c2_C<C>"), its shape, and mul, the lens_mul it is launched with (L = F * mul rows).  c2's acc is the
    ResBlock accumulation of hifigan/models.py:120-126 (1 = ADD, 2 = ADD_DIV by the number of ResBlocks on the last layer)."""
    sh = shapes or voc_shapes()
    out = [dict(kind="pre", B=B, L=F, mul=1, Cin=sh["n_mels"], Cout=sh["c0"], K=sh["pre_k"], dil=1, rate=1, act=0, res=0, acc=0)]
    L = F
    for s, u in enumerate(sh["ups"]):
        out.append(dict(kind="ups%d" % s, B=B, L=L, mul=L // F, Cin=u["cin"], Cout=u["rate"] * u["cout"], K=u["K"], dil=1, rate=u["rate"],
                        act=1, res=0, acc=0))
        L *= u["rate"]
        C, J = u["cout"], len(sh["res_k"])
        for j, K in enumerate(sh["res_k"]):
            D = len(sh["res_d"][j])
            for l, d in enumerate(sh["res_d"][j]):
                acc = 0 if (l < D - 1 or j == 0) else (2 if j == J - 1 else 1)
                out.append(dict(kind="c1_C%d" % C, B=B, L=L, mul=L // F, Cin=C, Cout=C, K=K, dil=d, rate=1, act=1, res=0, acc=0))
                out.append(dict(kind="c2_C%d" % C, B=B, L=L, mul=L // F, Cin=C, Cout=C, K=K, dil=1, rate=1, act=1, res=1, acc=acc))
    return out


def engine_launches(lib, B, F, mode, shapes=None, time_major=False):
    """Kernel launches of one ev_vocoder call at (B, F) in kernel mode `mode`, in order: plan keys
    (kernel, MODE, MT, KBG, BN, rate) for the tensor-core kernels, ("to_gp",), ("gp_sum_div",), ("conv_post",); in MODE FFMA
    ("transpose",) for a channels-first mel, ("conv1d_tm", TXN, NV, TM) per convolution and ("conv_post",)."""
    sh = shapes or voc_shapes()
    if mode == am_plans.FFMA:
        out = [] if time_major else [("transpose",)]
        for r in ffma_layers(B, F, sh):
            out.append(am_plans.conv1d_plan(lib, B, r["L"], r["Cin"], r["Cout"], r["K"], r["dil"])["key"])
        return out + [("conv_post",)]
    out = [("to_gp",), gp_plan(lib, B, F, sh["n_mels"], sh["c0"], sh["pre_k"], 1, 1, mode)["key"]]
    L = F
    for u in sh["ups"]:
        out.append(gp_plan(lib, B, L, u["cin"], u["rate"] * u["cout"], u["K"], 1, u["rate"], mode)["key"])
        L *= u["rate"]
        C, Ks, Ds = u["cout"], sh["res_k"], sh["res_d"]
        grp = _grouped_stage(lib, B, L, C, Ks, Ds, mode) if B * F <= GROUP_MAX_FRAMES else None
        if grp is not None:
            out += grp
            continue
        for j, K in enumerate(Ks):
            for d in Ds[j]:
                p = _fused(lib, B, L, C, K, d, mode)
                if p is not None:
                    out.append(p["key"])
                else:
                    out.append(gp_plan(lib, B, L, C, C, K, d, 1, mode)["key"])
                    out.append(gp_plan(lib, B, L, C, C, K, 1, 1, mode)["key"])
    out.append(("conv_post",))
    return out
