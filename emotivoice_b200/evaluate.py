"""Objective comparison of syntheses with recordings of the same sentences on the GPU (``ev_eval_compare``): mel-cepstral
distortion after dynamic time warping (DTW), F0 error and voicing error, per pair of a batch.

    from emotivoice_b200 import evaluate
    c = evaluate.compare(out["wav_predictions"][:, 0], recordings,
                         syn_lengths=[256 * int(n) for n in out["mel_lengths_host"]], ref_lengths=lens)
    c.mcd, c.f0_rmse, c.vuv_error, c.voiced_pairs, c.path_length      # (B,) device tensors, no host sync

Free-running synthesis predicts its own durations, so its frames do not line up with the recording's; the DTW path pairs them
before anything is measured.  Definitions, per pair, at 16 kHz (other rates are first resampled to 16 kHz):

1. Features.  L: the log-mel of ``feats.TacotronSTFT(1024, 256, 1024, 80, 16000, 0, 8000).mel_spectrogram``, ln of
   max(mel magnitude, 1e-5).  F0: ``feats.pitch_track(wav, 16000, 256, continuous=False)``, 0 for unvoiced frames.  An item
   of n samples has n // 256 + 1 frames of both: N frames for the synthesis, M for the recording.
2. Cepstra.  c_k[f] = (1/80) sum_{m=0..79} L[m, f] cos(pi k (m + 1/2) / 80), k = 1..24, in fp64: the products summed over m in
   ascending order, then divided by 80, the cosine table computed once on the host in fp64.  These are the cosine-series
   coefficients of the mel-band log-magnitude envelope without the level term c0, so a gain change moves only c0 (away from
   the 1e-5 clamp) and does not change the distance.
3. Local distance.  d(i, j) = sqrt(sum_{k=1..24} (c_k[i] - c'_k[j])^2), summed over ascending k, every product and sum
   rounded on its own (no fused multiply-add), correctly rounded square root.
4. DTW.  D(0,0) = d(0,0); D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)) over the predecessors that exist, ties to
   the first in that order (diagonal, then (i-1, j), then (i, j-1)).  The path is the backtrack from (N-1, M-1) to (0,0);
   its length P lies in [max(N, M), N + M - 1].
5. Statistics along the path, summed in path order from (0,0) in fp64.
   mcd = (10 sqrt(2) / ln 10) (1/P) sum d(i, j) in dB.  A frame is voiced iff its F0 > 0.  vuv_error: the share of pairs
   whose voicing differs.  voiced_pairs: the pairs voiced on both sides.  f0_rmse = sqrt(mean over those pairs of
   (1200 log2(f_syn / f_ref))^2) in cents, NaN when voiced_pairs = 0.

These cosine-series cepstra are this function's default (``cepstrum="mel"``); their values compare between runs of it.  For
the MCD papers report, pass ``cepstrum="world"``: step 2 then takes c1..c24 of the SPTK mel-cepstrum of WORLD's spectral
envelope, ``feats.sp2mc(feats.spectral_envelope(wav, 16000, 256, f0=F0), 24, alpha)`` with alpha = 0.42 by default (pyworld's
CheapTrick and pysptk's sp2mc restated on the GPU in fp64; not checked against pyworld or pysptk), from the same F0 track.
Steps 3 to 5 are unchanged.  The DTW is exact (no band, no fastdtw approximation), with the one step pattern above.  With
``cepstrum="mel"`` the cepstra, distances, DTW and path are bitwise ``oracle/eval_oracle.py``'s; with ``"world"`` the
distances, DTW and path are bitwise the oracle's on the GPU's mel-cepstra.  Every pair's results are the same bits whatever
else is in the batch and in which order.

Limits: each item holds at least ``feats.pitch_min_samples(16000)`` = 641 samples and at most 4096 frames at 16 kHz
(4096 * 256 - 1 samples, about 65.5 s).  The workspace holds d and a predecessor code for every cell of every pair, sized by
the batch's longest synthesis and longest recording: 9 B max(N) max(M) bytes, 151 MB per pair at 4096 x 4096, 4 GB for 1000
pairs of 10 s.  One long item thus costs every pair of its batch its size: evaluate a large test set in chunks of pairs of
similar length (sorted by length, say 32 to 128 pairs per call).  Forward only, no gradients.

No call waits for the device: lengths and tables go up through pinned memory, and the results stay on the device.  The first
call on a device builds its constant tables (the mel basis, the window, the cosine table; with ``"world"`` the sp2mc table of
each alpha) and allocates pinned host memory.
"""
import collections

import numpy as np
import torch

from . import _abi, audio, feats, recordings

SR = 16000
HOP = 256
N_MELS, N_CEPS = 80, 24
MAX_FRAMES = 4096
MIN_SAMPLES = feats.pitch_min_samples(SR)
MAX_SAMPLES = MAX_FRAMES * HOP - 1
WORLD_ALPHA = 0.42              # the all-pass constant MCD recipes use for 16 kHz speech

Comparison = collections.namedtuple("Comparison", "mcd f0_rmse vuv_error voiced_pairs path_length path")
Comparison.__doc__ = """Per-pair results of ``compare`` (device tensors of shape (B,)): mcd (dB), f0_rmse (cents) and vuv_error
(float64); voiced_pairs and path_length (int32); path: (B, P_max, 2) int32 pairs (syn frame, ref frame) from (0,0), -1 past
each pair's own path, P_max = max(N) + max(M) - 1 over the batch (the longest synthesis and the longest recording may be in
different rows); None unless asked for."""


def cos_table():
    """(24, 80) float64: row k - 1 holds cos(pi k (m + 1/2) / 80), m = 0..79."""
    k = np.arange(1, N_CEPS + 1, dtype=np.float64)[:, None]
    m = np.arange(N_MELS, dtype=np.float64)[None, :]
    return np.cos(np.pi * k * (m + 0.5) / N_MELS)


def _features(wav, lens):
    """16 kHz (B, L) items -> (log-mel (B, 80, F) float32, F0 (B, F) float64), frames per item n // 256 + 1: the mel of
    TacotronSTFT(1024, 256, 1024, 80, 16000, 0, 8000) without its range check."""
    bands = feats.mel_bands(SR, N_MELS, 0.0, 8000.0, wav.device)
    window = feats.scipy_hann(wav.device)
    mel, _, _ = feats.stft_features(wav, 1024 // 2, HOP, window, 0.0, bands=bands, lengths=lens, check_range=False)
    f0 = feats.pitch_track(wav, SR, HOP, continuous=False, lengths=lens)
    assert mel.shape[2] == f0.shape[1] == wav.shape[1] // HOP + 1, (tuple(mel.shape), tuple(f0.shape))
    assert all(feats.pitch_frames(n, SR, HOP) == n // HOP + 1 for n in lens)
    return mel, f0


def _check_cepstrum(cepstrum, alpha):
    """-> the alpha of ``cepstrum="world"`` (None for "mel"); ValueError for an unknown kind, alpha with "mel", |alpha| >= 1."""
    if cepstrum == "mel":
        if alpha is not None:
            raise ValueError("alpha applies to cepstrum='world' only")
        return None
    if cepstrum != "world":
        raise ValueError("cepstrum must be 'mel' or 'world', got %r" % (cepstrum,))
    alpha = WORLD_ALPHA if alpha is None else alpha
    feats._check_sp2mc(N_CEPS, alpha)
    return float(alpha)


def _world_features(wav, lens, table):
    """16 kHz (B, L) items -> (c1..c24 (B, F, 24) float64 of sp2mc(CheapTrick envelope), F0 (B, F) float64), F = L // 256 + 1:
    one F0 track feeds both the envelope and the statistics."""
    f0 = feats.pitch_track(wav, SR, HOP, continuous=False, lengths=lens)
    _, cep = feats.envelope_features(wav, SR, HOP, f0=f0, lengths=lens, table=table, envelope=False)
    return cep, f0


@torch.no_grad()
def compare(syn, ref, sample_rate=16000, syn_lengths=None, ref_lengths=None, return_path=False, cepstrum="mel", alpha=None):
    """Compares row b of ``syn`` with row b of ``ref`` (see the module docstring for the definitions).

    ``syn``, ``ref``: CUDA (B, L_syn) and (B, L_ref) float32 tensors.  ``sample_rate``: the rate of both, one ``audio.plan``
    accepts; other rates than 16 kHz are resampled to 16 kHz first (``ev_format_audio``, as ``resample_poly``).
    ``syn_lengths``, ``ref_lengths``: the valid samples of each row (a sequence or a CPU tensor of B integers); None: the whole
    row.  Each item must hold 641 to 4096 * 256 - 1 samples once at 16 kHz.  ``return_path``: also return the DTW paths.
    ``cepstrum``: "mel" (the log-mel's cosine series) or "world" (the SPTK mel-cepstrum of WORLD's envelope, warped by
    ``alpha``, 0.42 by default, |alpha| < 1; alpha is for "world" only).

    Returns a ``Comparison`` of device tensors, with no host sync.  The workspace grows with B max(N) max(M): batch long
    test sets in chunks of similar lengths (module docstring).  Invalid arguments raise ValueError before anything is
    enqueued."""
    alpha = _check_cepstrum(cepstrum, alpha)
    syn = recordings.recording_batch(syn, "syn")
    ref = recordings.recording_batch(ref, "ref")
    B = int(syn.shape[0])
    if int(ref.shape[0]) != B:
        raise ValueError("syn and ref must hold the same number of recordings, got %d and %d" % (B, int(ref.shape[0])))
    if syn.device != ref.device:
        raise ValueError("syn and ref must be on the same device")
    rate, up, down = audio.plan(sample_rate, "float32", SR)
    ls = recordings.host_lengths(syn_lengths, B, int(syn.shape[1]), "syn_lengths")
    lr = recordings.host_lengths(ref_lengths, B, int(ref.shape[1]), "ref_lengths")
    if rate != SR:                                # up / down take 16 kHz to the rate, so the way back is down / up
        ls16 = [audio.resampled_length(n, down, up) for n in ls]
        lr16 = [audio.resampled_length(n, down, up) for n in lr]
    else:
        ls16, lr16 = ls, lr
    for name, lens in (("syn", ls16), ("ref", lr16)):
        bad = [n for n in lens if not MIN_SAMPLES <= n <= MAX_SAMPLES]
        if bad:
            raise ValueError("each %s item must hold %d to %d samples at 16 kHz (at most %d frames), got %d"
                             % (name, MIN_SAMPLES, MAX_SAMPLES, MAX_FRAMES, bad[0]))
    if not isinstance(return_path, (bool, np.bool_)):
        raise ValueError("return_path must be True or False, got %r" % (return_path,))
    lib = _abi.load()
    dev = syn.device
    if rate != SR:
        syn, ls = recordings.resample(syn, ls, rate, SR)
        ref, lr = recordings.resample(ref, lr, rate, SR)
    assert ls == ls16 and lr == lr16
    if cepstrum == "world":
        table = feats.mcep_table(feats.world_fft_size(SR), N_CEPS, alpha, dev, first=1)
        (cep_s, f0_s), (cep_r, f0_r) = _world_features(syn, ls, table), _world_features(ref, lr, table)
    else:
        mel_s, f0_s = _features(syn, ls)
        mel_r, f0_r = _features(ref, lr)
    ns = [n // HOP + 1 for n in ls]
    nr = [n // HOP + 1 for n in lr]
    counts_in, (p_ns, p_nr) = recordings.upload([ns, nr], dev, np.int32)
    max_n, max_m = max(ns), max(nr)
    stats = torch.empty((3, B), dtype=torch.float64, device=dev)
    counts = torch.empty((2, B), dtype=torch.int32, device=dev)
    p_max = max_n + max_m - 1                     # the path stride ev_eval_compare takes: no pair's path is longer
    path = torch.empty((B, p_max, 2), dtype=torch.int32, device=dev) if return_path else None
    nb = int(lib.ev_eval_workspace_bytes(B, max_n, max_m))
    ws = torch.empty((nb,), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    if cepstrum == "world":
        _abi.check(lib.ev_eval_align(cep_s.data_ptr(), f0_s.data_ptr(), int(cep_s.shape[1]), p_ns, max_n, cep_r.data_ptr(),
                                     f0_r.data_ptr(), int(cep_r.shape[1]), p_nr, max_m, B, stats.data_ptr(), counts.data_ptr(),
                                     None if path is None else path.data_ptr(), p_max, ws.data_ptr(), nb, stream))
        return Comparison(stats[0], stats[1], stats[2], counts[0], counts[1], path)
    table = recordings.device_table("cos_table", cos_table, dev)
    _abi.check(lib.ev_eval_compare(mel_s.data_ptr(), f0_s.data_ptr(), int(mel_s.shape[2]), p_ns, max_n,
                                   mel_r.data_ptr(), f0_r.data_ptr(), int(mel_r.shape[2]), p_nr, max_m, B,
                                   table.data_ptr(), stats.data_ptr(), counts.data_ptr(),
                                   None if path is None else path.data_ptr(), p_max, ws.data_ptr(), nb, stream))
    return Comparison(stats[0], stats[1], stats[2], counts[0], counts[1], path)
