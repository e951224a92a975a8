"""ctypes binding of libemotivoice_b200.so (include/emotivoice_b200.h).

The shared library is the only compute path of this package.  If it is missing or fails
to load this module raises -- there is deliberately no CPU / eager-PyTorch fallback.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libemotivoice_b200.so")

EV_OK = 0
EV_ENOWEIGHT = -2
EV_EPELEN = -5
ACT_NONE, ACT_LRELU, ACT_RELU, ACT_GELU, ACT_TANH = 0, 1, 2, 3, 4
ACC_STORE, ACC_ADD, ACC_ADD_DIV = 0, 1, 2
PREC_FP32, PREC_TF32, PREC_FP32_FFMA, PREC_BF16 = 0, 1, 2, 3
PRECISIONS = {"fp32": PREC_FP32, "tf32": PREC_TF32, "fp32_ffma": PREC_FP32_FFMA, "bf16": PREC_BF16}


class EvConfig(ctypes.Structure):
    """ev_config (include/emotivoice_b200.h)."""
    _fields_ = [
        ("n_vocab", ctypes.c_int32), ("n_speaker", ctypes.c_int32),
        ("hidden", ctypes.c_int32), ("n_heads", ctypes.c_int32),
        ("enc_layers", ctypes.c_int32), ("dec_layers", ctypes.c_int32),
        ("ffn_kernel", ctypes.c_int32), ("bert_dim", ctypes.c_int32),
        ("dur_layers", ctypes.c_int32), ("pitch_layers", ctypes.c_int32), ("energy_layers", ctypes.c_int32),
        ("pred_kernel", ctypes.c_int32), ("embed_kernel", ctypes.c_int32), ("n_mels", ctypes.c_int32),
        ("voc_c0", ctypes.c_int32), ("n_ups", ctypes.c_int32),
        ("up_rates", ctypes.c_int32 * 8), ("up_kernels", ctypes.c_int32 * 8),
        ("n_resk", ctypes.c_int32), ("res_kernels", ctypes.c_int32 * 4),
        ("n_dil", ctypes.c_int32), ("res_dils", (ctypes.c_int32 * 4) * 4),
    ]


class EvStyleConfig(ctypes.Structure):
    """ev_style_config (include/emotivoice_b200.h)."""
    _fields_ = [(n, ctypes.c_int32) for n in ("vocab_size", "max_position", "type_vocab", "hidden", "n_heads", "n_layers",
                                              "intermediate", "n_head_out")]


class EvError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libemotivoice_b200 error %d: %s" % (code, msg))
        self.code = code


_vp, _i, _f, _sz, _u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_uint64

# name -> (restype, argtypes); must list every EV_API symbol of the header (tests check this)
SIGNATURES = {
    "ev_abi_version": (_i, []),
    "ev_last_error": (ctypes.c_char_p, []),
    "ev_create": (_i, [ctypes.POINTER(_vp), _i, ctypes.POINTER(EvConfig)]),
    "ev_destroy": (None, [_vp]),
    "ev_bind_weights": (_i, [_vp, _vp, _sz, _vp, _i]),
    "ev_bind_pe": (_i, [_vp, _vp, _i]),
    "ev_phase1_workspace_bytes": (_sz, [_vp, _i, _i]),
    "ev_phase2_workspace_bytes": (_sz, [_vp, _i, _i]),
    "ev_am_phase1": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_am_phase1_prosody": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_am_phase1_controls": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _sz, _vp]),
    "ev_am_phase2": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "ev_vocoder": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "ev_join_mel": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "ev_wav_to_pcm16": (_i, [_vp, _vp, _sz, _vp]),
    "ev_format_audio": (_i, [_vp, ctypes.c_longlong, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "ev_loudness_workspace_bytes": (_sz, [_i, ctypes.c_longlong, _i]),
    "ev_loudness": (_i, [_vp, ctypes.c_longlong, _vp, _vp, _i, _i, _vp, _f, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_limit_workspace_bytes": (_sz, [_i, ctypes.c_longlong, _i]),
    "ev_limit": (_i, [_vp, ctypes.c_longlong, _vp, _vp, _i, _i, _vp, _vp, _f, _f, _vp, _i, _i, _i, _i, ctypes.c_double, _vp,
                      ctypes.c_longlong, _vp, _sz, _vp]),
    "ev_meter_workspace_bytes": (_sz, [_i, ctypes.c_longlong, _i]),
    "ev_meter": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, ctypes.c_longlong, _vp, _sz, _vp]),
    "ev_eval_workspace_bytes": (_sz, [_i, _i, _i]),
    "ev_eval_compare": (_i, [_vp, _vp, ctypes.c_longlong, _vp, _i, _vp, _vp, ctypes.c_longlong, _vp, _i, _i, _vp, _vp, _vp, _vp,
                             ctypes.c_longlong, _vp, _sz, _vp]),
    "ev_eval_align": (_i, [_vp, _vp, ctypes.c_longlong, _vp, _i, _vp, _vp, ctypes.c_longlong, _vp, _i, _i, _vp, _vp, _vp,
                           ctypes.c_longlong, _vp, _sz, _vp]),
    "ev_flac_bound_bytes": (_sz, [ctypes.c_longlong]),
    "ev_flac_workspace_bytes": (_sz, [_i, ctypes.c_longlong]),
    "ev_flac_encode": (_i, [_vp, _vp, _i, _vp, _i, _vp, _sz, _vp, _vp, _sz, _vp]),
    "ev_watermark_embed": (_i, [_vp, ctypes.c_longlong, _vp, _vp, _i, _i, _u64, _vp, ctypes.c_longlong, _vp]),
    "ev_watermark_detect_workspace_bytes": (_sz, [_i]),
    "ev_watermark_detect": (_i, [_vp, ctypes.c_longlong, _vp, _i, _u64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_launch_count": (_u64, []),
    "ev_op_conv1d": (_i, [_vp, _vp, _vp, _sz, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _f, _i, _i, _f, _vp]),
    "ev_op_conv1d_tc": (_i, [_vp, _vp, _i, _vp, _sz, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _f, _i, _i, _f, _vp, _sz, _vp]),
    "ev_op_conv1d_tc_ks": (_i, [_vp, _vp, _i, _vp, _sz, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _f, _i, _i, _f, _i, _vp, _sz, _vp]),
    "ev_set_precision": (_i, [_vp, _i]),
    "ev_op_conv1d_gp": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _f, _i, _f, _vp]),
    "ev_op_resblock_gp": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _i, _i, _f, _vp]),
    "ev_debug_resblock_gp_plan": (_i, [_i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_op_conv1d_gp_group": (_i, [_i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _f, _vp]),
    "ev_op_resblock_gp_group": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "ev_debug_resblock_gp_group_plan": (_i, [_i, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_op_gp_sum_div": (_i, [_vp, _vp, _vp, _vp, _sz, _f, _vp]),
    "ev_debug_gp_group_plan": (_i, [_i, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_debug_gp_plan": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_op_to_gp": (_i, [_vp, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_longlong, _vp, _i, _i, _i, _i, _vp]),
    "ev_op_conv_post_gp": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp]),
    "ev_debug_tc_plan": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_debug_conv1d_plan": (_i, [_i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int)]),
    "ev_op_conv_post": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp]),
    "ev_op_layernorm": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    "ev_op_attention": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ev_op_attention_tc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "ev_op_gauss_upsample": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ev_op_duration_scan": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "ev_op_duration_scan_controls": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "ev_op_gauss_upsample_centers": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "ev_op_layernorm_embed": (_i, [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "ev_op_cond_bias": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "ev_op_rowdot": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "ev_op_mask_rows": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "ev_op_var_embed_add": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ev_op_bert_embed_ln": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "ev_op_row_gemv": (_i, [_vp, _sz, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ev_op_mas": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_op_average_by_duration": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "ev_op_align_logp": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "ev_op_get_segments": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "ev_stft_features": (_i, [_vp, ctypes.c_longlong, _vp, _i, _i, _i, _i, _vp, _vp, _f, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "ev_pitch_workspace_bytes": (_sz, [_i, ctypes.c_longlong, _i, ctypes.c_double, _i]),
    "ev_pitch": (_i, [_vp, ctypes.c_longlong, _vp, _i, _i, ctypes.c_double, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ev_world_envelope": (_i, [_vp, ctypes.c_longlong, _vp, _i, _i, ctypes.c_double, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "ev_sp2mc": (_i, [_vp, ctypes.c_longlong, _i, _vp, _i, _vp, _vp]),
    "ev_style_create": (_i, [ctypes.POINTER(_vp), _i, ctypes.POINTER(EvStyleConfig)]),
    "ev_style_destroy": (None, [_vp]),
    "ev_style_bind_weights": (_i, [_vp, _vp, _sz, _vp, _i]),
    "ev_style_set_precision": (_i, [_vp, _i]),
    "ev_style_workspace_bytes": (_sz, [_vp, _i, _i]),
    "ev_style_forward": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
}

_lib = None


def load():
    """dlopen the engine (once).  Raises if the library has not been built:
    run ``python -m emotivoice_b200.build`` (or ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libemotivoice_b200.so not found at %s -- build it with `python -m emotivoice_b200.build`. "
            "There is no CPU fallback for this engine." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.ev_abi_version() != 1:
        raise RuntimeError("libemotivoice_b200.so ABI version %d != 1" % lib.ev_abi_version())
    _lib = lib
    return lib


def check(rc):
    if rc != EV_OK:
        raise EvError(rc, load().ev_last_error().decode(errors="replace"))


def launch_count():
    return int(load().ev_launch_count())


def make_config(conf):
    """attr-config (config.yaml model.* names) -> ev_config."""
    m = conf.model
    c = EvConfig()
    if not (m.encoder_n_hidden == m.decoder_n_hidden == m.variance_n_hidden):
        raise ValueError("engine requires encoder/decoder/variance hidden sizes to be equal")
    if m.encoder_n_heads != m.decoder_n_heads or m.encoder_kernel_size_conv_mod != m.decoder_kernel_size_conv_mod:
        raise ValueError("engine requires encoder and decoder to share heads / conv kernel size")
    if m.duration_kernel_size != m.variance_kernel_size or m.variance_kernel_size != 3:
        raise ValueError("engine requires duration/variance kernel size 3 (energy predictor is hard-coded to 3)")
    if str(m.resblock) != "1":
        raise ValueError("only ResBlock1 generators are supported (config.yaml:87)")
    c.n_vocab, c.n_speaker = int(conf.n_vocab), int(conf.n_speaker)
    c.hidden, c.n_heads = int(m.encoder_n_hidden), int(m.encoder_n_heads)
    c.enc_layers, c.dec_layers = int(m.encoder_n_layers), int(m.decoder_n_layers)
    c.ffn_kernel, c.bert_dim = int(m.encoder_kernel_size_conv_mod), int(m.bert_embedding)
    c.dur_layers, c.pitch_layers, c.energy_layers = int(m.duration_n_layers), int(m.variance_n_layers), 2
    c.pred_kernel, c.embed_kernel = int(m.variance_kernel_size), int(m.variance_embed_kernel_size)
    c.n_mels, c.voc_c0 = int(conf.n_mels), int(m.upsample_initial_channel)
    if int(m.initial_channel) != int(conf.n_mels):
        raise ValueError("initial_channel must equal n_mels")
    c.n_ups = len(m.upsample_rates)
    for i, (u, k) in enumerate(zip(m.upsample_rates, m.upsample_kernel_sizes)):
        c.up_rates[i], c.up_kernels[i] = int(u), int(k)
    c.n_resk = len(m.resblock_kernel_sizes)
    c.n_dil = len(m.resblock_dilation_sizes[0])
    for j, k in enumerate(m.resblock_kernel_sizes):
        c.res_kernels[j] = int(k)
        if len(m.resblock_dilation_sizes[j]) != c.n_dil:
            raise ValueError("all ResBlocks must have the same number of dilations")
        for l, d in enumerate(m.resblock_dilation_sizes[j]):
            c.res_dils[j][l] = int(d)
    return c
