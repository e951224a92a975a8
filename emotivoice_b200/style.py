"""Host-side mirror of the reference's style encoder boundary (SURVEY.md s8f rank 1).

``StyleEncoder`` has the reference's class name, constructor argument, state-dict keys and ``forward`` signature
(models/prompt_tts_modified/simbert.py:33-72), so the callers' plumbing runs unchanged
(inference_am_vocoder_joint.py:25-38,59-65: ``StyleEncoder(config)``, ``load_state_dict(ckpt, strict=False)``,
``style_encoder(input_ids=..., token_type_ids=..., attention_mask=...)["pooled_output"]``) -- except that it lives on the
GPU (``.to(device)``), where one pass costs microseconds instead of the two CPU BERT passes per utterance of the reference.

The module is a parameter tree only; every FLOP of ``forward`` runs in libemotivoice_b200.so (``ev_style_forward``).
Tokenisation stays with the caller (it needs the checkpoint's vocabulary file).  No CPU path.
"""
import ctypes
import json
import os

import torch

from . import _abi, packing, synth
from .modules import _EngineOwner, _prep, _register

_BERT_KEYS = ("vocab_size", "hidden_size", "num_hidden_layers", "num_attention_heads", "intermediate_size",
              "max_position_embeddings", "type_vocab_size")


def _style_arch(config, bert_config):
    """Architecture integers: the reference takes them from the checkpoint's config.json via ``AutoModel.from_pretrained``
    (simbert.py:37).  Here: ``bert_config`` (attr object or dict with BertConfig names) > ``<config.bert_path>/config.json``
    when that is a local directory > simbert-base-chinese's published dimensions."""
    sc = synth.style_config(False)
    src = None
    if bert_config is not None:
        src = bert_config if isinstance(bert_config, dict) else {k: getattr(bert_config, k) for k in _BERT_KEYS if hasattr(bert_config, k)}
    else:
        path = getattr(config, "bert_path", None)
        if isinstance(path, str) and os.path.isfile(os.path.join(path, "config.json")):
            with open(os.path.join(path, "config.json")) as f:
                src = json.load(f)
    if src:
        for k in _BERT_KEYS:
            if k in src:
                sc[k] = int(src[k])
        if src.get("hidden_act", "gelu") != "gelu" or src.get("position_embedding_type", "absolute") != "absolute":
            raise NotImplementedError("style encoder: only gelu / absolute-position BERT checkpoints are supported")
    for n in packing.STYLE_HEADS:
        if hasattr(config, n + "_n_labels"):
            sc[n + "_n_labels"] = int(getattr(config, n + "_n_labels"))
    if hasattr(config, "style_dim"):
        sc.style_dim = int(config.style_dim)
    if hasattr(config, "bert_hidden_size") and int(config.bert_hidden_size) != sc.hidden_size:
        raise ValueError("config.bert_hidden_size=%s but the BERT hidden size is %d" % (config.bert_hidden_size, sc.hidden_size))
    return sc


def _drop_position_ids(module, state_dict, prefix, *args):
    """Checkpoints written with transformers < 4.31 carry the ``position_ids`` arange as a persistent buffer."""
    state_dict.pop(prefix + "bert.embeddings.position_ids", None)


class _StyleEngine:
    """One ev_style_ctx + its packed weight blob on one device."""

    def __init__(self, sc, packed, device, precision):
        self.lib = _abi.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("emotivoice_b200 runs on CUDA (sm_90a) only; got device %s. There is no CPU fallback." % (self.device,))
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        _, self.n_head_out = packing.style_head_slices(sc)
        self.cfg = _abi.EvStyleConfig(sc.vocab_size, sc.max_position_embeddings, sc.type_vocab_size, sc.hidden_size,
                                      sc.num_attention_heads, sc.num_hidden_layers, sc.intermediate_size, self.n_head_out)
        handle = ctypes.c_void_p()
        _abi.check(self.lib.ev_style_create(ctypes.byref(handle), idx, ctypes.byref(self.cfg)))
        self.handle = handle
        blob, self.index = packing.make_blob(packed)
        self.blob = blob.to(self.device)
        _abi.check(self.lib.ev_style_bind_weights(self.handle, self.blob.data_ptr(), self.blob.numel(),
                                                  ctypes.cast(self.index, ctypes.c_void_p), len(self.index)))
        self.set_precision(precision)

    def set_precision(self, precision):
        if precision not in ("fp32", "tf32"):
            raise ValueError("style encoder precision must be 'fp32' (3xTF32) or 'tf32'")
        _abi.check(self.lib.ev_style_set_precision(self.handle, _abi.PRECISIONS[precision]))
        self.precision = precision

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.ev_style_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def forward(self, ids, tts, lens):
        B, N = ids.shape
        H = int(self.cfg.hidden)
        dev = self.device
        pooled = torch.empty((B, H), dtype=torch.float32, device=dev)
        heads = torch.empty((B, self.n_head_out), dtype=torch.float32, device=dev)
        n = int(self.lib.ev_style_workspace_bytes(self.handle, B, N))
        ws = torch.empty((n,), dtype=torch.uint8, device=dev)
        _abi.check(self.lib.ev_style_forward(self.handle, ids.data_ptr(), tts.data_ptr(), lens.data_ptr(), B, N, pooled.data_ptr(),
                                             heads.data_ptr(), ws.data_ptr(), n, torch.cuda.current_stream(dev).cuda_stream))
        return pooled, heads


class StyleEncoder(_EngineOwner):
    """simbert.py:33-72.  ``config`` is the reference's global Config (``bert_path``, ``bert_hidden_size``, ``*_n_labels``,
    ``style_dim``); ``bert_config`` optionally gives the BERT dimensions (see ``_style_arch``)."""

    def __init__(self, config, bert_config=None, _init=None):
        super().__init__()
        self.config = config
        self.arch = _style_arch(config, bert_config)
        if _init is None:
            seed = int(torch.randint(0, 2 ** 31 - 1, ()).item())
            _init = synth.make_style_state_dict(self.arch, seed=seed)
        for k, v in _init.items():
            _register(self, k, v.clone())
        self._register_load_state_dict_pre_hook(_drop_position_ids, with_module=True)

    @property
    def precision(self):
        """"fp32" (default): fp32-accurate 3xTF32 on the tensor cores; "tf32": one tf32 MMA per K step."""
        return self._ev_precision

    @precision.setter
    def precision(self, value):
        if value not in ("fp32", "tf32"):
            raise ValueError("style encoder precision must be 'fp32' or 'tf32'")
        self._ev_precision = value
        if self._ev_engine is not None:
            self._ev_engine.set_precision(value)

    def _engine(self):
        eng = self._ev_engine
        dev = next(self.parameters()).device
        if eng is not None and not self._ev_dirty and eng.device == dev:
            return eng
        with self._ev_lock:
            if self._ev_engine is None or self._ev_dirty or self._ev_engine.device != dev:
                self._ev_engine = _StyleEngine(self.arch, packing.pack_style_state_dict(self.state_dict(), self.arch), dev,
                                               self._ev_precision)
                self._ev_dirty = False
            return self._ev_engine

    @torch.no_grad()
    def forward(self, input_ids, token_type_ids, attention_mask):
        eng = self._engine()
        dev = eng.device
        ids = _prep(input_ids, torch.int64, dev)
        tts = _prep(token_type_ids, torch.int64, dev)
        mask = _prep(attention_mask, torch.int64, dev)
        if ids.dim() != 2 or tts.shape != ids.shape or mask.shape != ids.shape:
            raise RuntimeError("shape mismatch: input_ids %s, token_type_ids %s, attention_mask %s"
                               % (tuple(ids.shape), tuple(tts.shape), tuple(mask.shape)))
        lens = mask.sum(dim=1)
        # one host round trip validates what the library would otherwise read out of bounds / mis-mask; the tokenizer's
        # padding is always a suffix (inference_am_vocoder_joint.py:25-29 never pads at all: one prompt per call)
        prefix = (torch.arange(ids.shape[1], device=dev)[None, :] < lens[:, None]).to(torch.int64)
        bad = torch.stack([(mask != prefix).any(), (lens < 1).any(), (ids < 0).any() | (ids >= self.arch.vocab_size).any(),
                           (tts < 0).any() | (tts >= self.arch.type_vocab_size).any()]).tolist()
        if bad[0] or bad[1]:
            raise RuntimeError("attention_mask must be a non-empty prefix of ones per item (right padding)")
        if bad[2] or bad[3]:
            raise IndexError("input_ids / token_type_ids out of range of the embedding tables")
        if ids.shape[1] > self.arch.max_position_embeddings:
            raise RuntimeError("sequence length %d exceeds max_position_embeddings=%d" % (ids.shape[1], self.arch.max_position_embeddings))
        pooled, heads = eng.forward(ids, tts, lens.contiguous())
        slices, _ = packing.style_head_slices(self.arch)
        out = {"pooled_output": pooled}
        for n in ("pitch", "speed", "energy", "emotion"):          # key order of simbert.py:64-71
            c0, k = slices[n]
            out[n + "_outputs"] = heads[:, c0:c0 + k]
        return out
