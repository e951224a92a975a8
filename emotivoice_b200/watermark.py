"""Finds the watermark ``format_audio(watermark=KEY)`` embeds: ``detect(wav, sample_rate, key)`` answers "does this recording
carry the mark of this key?" for each recording of a batch, on the GPU (``ev_watermark_detect``).

The mark carries no payload.  At 16 kHz, in MCLT frames of 1024 samples (hop 512, sine window), each MDCT coefficient C of
bins 19..217 (about 300-3400 Hz) of frame j was changed by alpha * M * s(key, j mod 64, k), M the MCLT magnitude and s = +-1
a keyed pattern (``audio.WATERMARK_*``).  The detector analyses the recording on the grid shifted by tau samples for every tau
in [0, 512), takes u = C / M in the band (skipping cells with M = 0), folds the frames modulo 64 into b[tau, r, k], and for
every frame phase m0 in [0, 64) computes

    z(tau, m0) = sum_{r,k} s(key, (r + m0) mod 64, k) b[tau, r, k] / sqrt(sum_{r,k} b[tau, r, k]^2).

It reports the largest z of each recording and its (tau, m0): for a recording that starts c samples into a marked output,
tau = -c mod 512 and m0 = ((c + tau) / 512) mod 64.

False positives.  Take a recording and a key chosen independently of it, and model the pattern as an ideal keyed PRF: the
signs s(key, ., .) are then independent fair +-1 given b, and for a fixed (tau, m0) they multiply 64 * 199 distinct cells of
b.  The numerator is a Rademacher sum sum_i s_i b_i, and Hoeffding's inequality gives P(sum_i s_i b_i >= t ||b||) <=
exp(-t^2 / 2), with no Gaussian assumption and whatever the recording.  A union over the 512 * 64 = 32768 hypotheses gives
P(max z >= t) <= 32768 exp(-t^2 / 2); at t = DETECT_Z = 7.0 that is 32768 * e^-24.5 = 7.6e-7 per (recording, key).  SplitMix64
is not a cryptographic PRF, so the bound is for keys chosen without knowledge of the recording.

Silence (every cell M = 0) gives z = 0.
"""
import torch

from . import _abi, audio, recordings

DETECT_Z = audio.WATERMARK_DETECT_Z
SR = 16000


@torch.no_grad()
def detect(wav, sample_rate, key, lengths=None):
    """Searches each recording for the mark of ``key``.

    ``wav``: a CUDA (B, L) float32 tensor, one recording per row.  ``sample_rate``: their rate in Hz, at least 8000; a rate
    other than 16 kHz is first resampled to 16 kHz by ``ev_format_audio`` (the rates ``audio.plan`` accepts).  ``key``: an
    integer in [1, 2^63 - 1].  ``lengths``: the valid samples of each row (a sequence or a CPU tensor of B integers in [0, L]);
    None: every row is L samples.

    Returns (z float32, offset int32, phase int32) device tensors of shape (B,): the largest z of each recording and its grid
    offset tau and frame phase m0.  z >= DETECT_Z means the mark is present (see the module docstring for the bound).  No
    sync.  Invalid arguments raise ValueError before anything is enqueued."""
    wav = recordings.recording_batch(wav)
    B, L = wav.shape
    rate = audio.plan(sample_rate, "float32", SR)[0]
    if rate < audio.WATERMARK_MIN_RATE:
        raise ValueError("the mark's band needs a rate of at least %d Hz, got %d" % (audio.WATERMARK_MIN_RATE, rate))
    key = audio.check_watermark(key)
    lens = recordings.host_lengths(lengths, B, L)
    lib = _abi.load()
    dev = wav.device
    if rate != SR:
        wav, lens = recordings.resample(wav, lens, rate, SR)
    n = recordings.upload([lens], dev)[0]
    z = torch.empty((B,), dtype=torch.float32, device=dev)
    offset = torch.empty((B,), dtype=torch.int32, device=dev)
    phase = torch.empty((B,), dtype=torch.int32, device=dev)
    nb = int(lib.ev_watermark_detect_workspace_bytes(B))
    ws = torch.empty((nb,), dtype=torch.uint8, device=dev)
    _abi.check(lib.ev_watermark_detect(wav.data_ptr(), int(wav.stride(0)), n.data_ptr(), B, key, z.data_ptr(), offset.data_ptr(),
                                       phase.data_ptr(), ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    return z, offset, phase
