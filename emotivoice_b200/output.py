"""The output chain of one engine: the watermark (ev_watermark_embed), loudness measurement (ev_loudness), true-peak limiting
(ev_limit), resampling and encoding (ev_format_audio) and FLAC (ev_flac_encode) of a forward's outputs, in that order, with
the filter banks and coefficients those stages read, and the loudness meter (ev_meter) of what it delivers.
``JETSGenerator.format_audio`` / ``measure_loudness`` / ``meter`` validate their arguments and call it under the engine's lock.
"""
import numpy as np
import torch

from . import _abi, audio, loudness, recordings

_DTYPES = {"float32": torch.float32, "pcm16": torch.int16, "mulaw": torch.uint8, "alaw": torch.uint8}


class Chain:
    """The output stages of the engine on ``device``; ``ws(kind, nbytes)`` is the engine's workspace arena."""

    def __init__(self, device, lib, ws):
        self.device, self.lib, self._ws = device, lib, ws

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _loudness(self, wav, n_in_ptr, items_ptr, k, sr, target):
        """ev_loudness of the k listed items (device i64 n_in / items pointers) -> device (lufs, peak, gain) float32 (k,)."""
        res = torch.empty((3, k), dtype=torch.float32, device=self.device)
        stride = int(wav.stride(0))
        ws = self._ws("loudness", self.lib.ev_loudness_workspace_bytes(k, stride, sr))
        _abi.check(self.lib.ev_loudness(wav.data_ptr(), stride, n_in_ptr, items_ptr, k, sr, loudness.k_weighting(sr).data_ptr(),
                                        float(target), res[0].data_ptr(), res[1].data_ptr(), res[2].data_ptr(), ws.data_ptr(),
                                        ws.numel(), self._stream()))
        return res[0], res[1], res[2]

    def _limit(self, wav, n_in_ptr, items_ptr, k, sr, rate, lufs0, lufs1, target, ceiling, out):
        """ev_limit of the k listed items into ``out`` (k, L) fp32, pre-gain 10^((target - L) / 20) of each given loudness."""
        bank, hold = recordings.device_table(("limit_bank", sr, rate), lambda: audio.limit_bank(sr, rate), self.device)
        L = audio.limit_lookahead(sr)
        stride = int(wav.stride(0))
        ws = self._ws("limit", self.lib.ev_limit_workspace_bytes(k, stride, L))
        _abi.check(self.lib.ev_limit(wav.data_ptr(), stride, n_in_ptr, items_ptr, k, sr, None if lufs0 is None else lufs0.data_ptr(),
                                     None if lufs1 is None else lufs1.data_ptr(), float(-23.0 if target is None else target),
                                     float(ceiling), bank.data_ptr(), int(bank.shape[0]), int(bank.shape[1]), L, hold,
                                     audio.limit_release(sr), out.data_ptr(), int(out.stride(0)), ws.data_ptr(), ws.numel(),
                                     self._stream()))

    def measure(self, wav, n_in, items, sr):
        """ev_loudness: (B,1,L) fp32 waveform at ``sr`` Hz, host per-item valid samples and the listed items -> device
        (lufs, peak) float32 (len(items),)."""
        meta, (p_n, p_items) = recordings.upload([n_in, items], self.device)
        lufs, pk, _ = self._loudness(wav, p_n, p_items, len(items), sr, -23.0)      # any valid target: the gain is not used
        return lufs, pk

    def meter(self, packed, offs, rate, series):
        """ev_meter of the outputs ``format`` packed as float32 at ``rate`` Hz (a multiple of 10), output k at
        packed[offs[k]:offs[k + 1]] -> ``loudness.Meter``.  No sync."""
        lens = np.diff(offs).tolist()
        meta, (p_meta, _) = recordings.upload([offs[:-1], lens], self.device)
        if packed.numel() == 0:                  # every output is empty: ev_meter reads no sample, but needs an address
            packed = torch.empty((1,), dtype=torch.float32, device=self.device)
        return loudness.enqueue(packed.data_ptr(), p_meta, lens, rate, lambda nb: self._ws("meter", nb), series)

    def format(self, wav, n_in, items, fmt, sr):
        """The listed items of a (B,1,L) fp32 waveform at ``sr`` Hz, host valid samples ``n_in`` (B ints <= L), in the
        ``audio.OutputFormat`` ``fmt`` -> (packed device tensor, (len(items)+1,) int64 host offsets).

        With ``fmt.watermark``, ev_watermark_embed first writes the marked items to the "marked" workspace, and every later
        stage reads that instead of ``wav``, so loudness targets and the ceiling hold for what is delivered.
        With ``fmt.true_peak``, ev_limit then writes the limited items to the "limited" workspace, which the later stages read:
        with ``fmt.loudness`` two passes (L0 of the items, limit x * g1, L1 of that result, limit x * g1 * g2; see
        ``JETSGenerator.format_audio``), else one pass with no pre-gain.  Otherwise with ``fmt.loudness`` one ev_loudness gives
        the gain of ev_format_audio.  "flac" encodes the PCM16 result and reads its image offsets back: the only sync."""
        lib, k = self.lib, len(items)
        encoding = "pcm16" if fmt.encoding == audio.FLAC else fmt.encoding
        offs = audio.packed_offsets(n_in, items, fmt.up, fmt.down)
        packed = torch.empty((int(offs[-1]),), dtype=_DTYPES[encoding], device=self.device)
        if packed.numel() == 0:                  # every listed output is empty (never for "flac"): nothing to launch
            return packed, offs
        arrays = [n_in, items, offs]
        if fmt.true_peak is not None or fmt.watermark is not None:
            arrays.append([int(n_in[b]) for b in items])                 # the limited / marked items' lengths, in listed order
        meta, ptrs = recordings.upload(arrays, self.device)
        p_n, p_items, p_off = ptrs[:3]
        src, src_n, src_items, gain = wav, p_n, p_items, None
        stride = int(wav.stride(0))
        if fmt.watermark is not None:
            marked = self._ws("marked", 4 * k * stride)[:4 * k * stride].view(torch.float32).view(k, stride)
            _abi.check(lib.ev_watermark_embed(wav.data_ptr(), stride, p_n, p_items, k, sr, fmt.watermark, marked.data_ptr(), stride,
                                              self._stream()))
            src, src_n, src_items = marked, ptrs[3], None
        if fmt.true_peak is not None:
            p_nl = ptrs[3]
            lim = self._ws("limited", 4 * k * stride)[:4 * k * stride].view(torch.float32).view(k, stride)
            lufs0 = lufs1 = None
            if fmt.loudness is not None:
                lufs0 = self._loudness(src, src_n, src_items, k, sr, fmt.loudness)[0]
                self._limit(src, src_n, src_items, k, sr, fmt.rate, lufs0, None, fmt.loudness, fmt.true_peak, lim)
                lufs1 = self._loudness(lim, p_nl, None, k, sr, fmt.loudness)[0]
            self._limit(src, src_n, src_items, k, sr, fmt.rate, lufs0, lufs1, fmt.loudness, fmt.true_peak, lim)
            src, src_n, src_items = lim, p_nl, None
        elif fmt.loudness is not None:
            gain = self._loudness(src, src_n, src_items, k, sr, fmt.loudness)[2]
        bank = None
        if (fmt.up, fmt.down) != (1, 1):
            bank = recordings.polyphase_bank(fmt.up, fmt.down, self.device)
        _abi.check(lib.ev_format_audio(src.data_ptr(), int(src.stride(0)), src_n, src_items, k, p_off,
                                       None if bank is None else bank.data_ptr(), fmt.up, fmt.down,
                                       0 if bank is None else int(bank.shape[1]), audio.ENCODINGS[encoding], packed.data_ptr(),
                                       None if gain is None else gain.data_ptr(), self._stream()))
        if fmt.encoding != audio.FLAC:
            return packed, offs
        counts = np.ascontiguousarray(np.diff(offs), dtype=np.int64)
        bound = sum(int(lib.ev_flac_bound_bytes(int(n))) for n in counts)
        out = torch.empty((bound,), dtype=torch.uint8, device=self.device)
        out_off = torch.empty((k + 1,), dtype=torch.int64, device=self.device)
        ws = self._ws("flac", lib.ev_flac_workspace_bytes(k, int(counts.max())))
        _abi.check(lib.ev_flac_encode(packed.data_ptr(), p_off, k, counts.ctypes.data, int(fmt.rate), out.data_ptr(), bound,
                                      out_off.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()))
        host = torch.empty((k + 1,), dtype=torch.int64, pin_memory=True)
        host.copy_(out_off, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        flac_offs = host.numpy().copy()
        return out[:int(flac_offs[-1])], flac_offs
