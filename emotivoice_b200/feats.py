"""Log-mel spectrograms and frame energy of recordings on the GPU, with the reference's names and signatures:
``TacotronSTFT`` (models/prompt_tts_modified/tacotron_stft.py:46-80), ``mel_spectrogram_torch`` (mel_process.py:77-110),
``Energy`` (models/prompt_tts_modified/feats.py:159-213) and ``Pitch`` (feats.py:83-156), pyworld.dio + pyworld.stonemask
restated on the GPU in fp64 (``ev_pitch``, csrc/pitch_kernels.cu); and, with no reference counterpart, WORLD spectral
envelopes (``spectral_envelope``, pyworld.cheaptrick) and SPTK mel-cepstra (``sp2mc``, pysptk.sp2mc) in fp64 (``ev_world_envelope``,
``ev_sp2mc``, csrc/world_kernels.cu), the features of paper-style mel-cepstral distortion.

These are the features the reference's data preparation computes per utterance on the CPU: the mel targets the acoustic model
and the vocoder were trained on (prompt_dataset.py:29-49), the mel distance of its validation and training step
(train_am_vocoder_joint.py:99-118) and the energy targets (prompt_dataset.py:82-86).  All three are one launch of
``stft_feats_kernel`` (csrc/feats_kernels.cu): a fused 1024-point fp32 FFT per frame, magnitude, mel bands, log and energy.
They differ only in the padding, the magnitude's epsilon and the rounding of the Hann window, which each passes its own.

librosa, which the reference uses for the mel basis and the energy's STFT, is not a dependency: ``mel_filterbank`` restates
``librosa.filters.mel`` (Slaney scale and norm) and is checked against torchaudio's ``melscale_fbanks``.  Inputs and outputs are
CUDA tensors; forward only (no gradients), FFT size 1024 only.
"""
import numpy as np
import torch
import torch.nn as nn

from . import _abi, recordings

N_FFT = 1024
_MAX_MELS = 128
_STATUS_RANGE = 1               # ev_stft_features: a sample outside [-1, 1]


def _check(t, name):
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise RuntimeError("%s must be a CUDA tensor: emotivoice_b200 has no CPU path" % name)


def _hz_to_mel(frequencies):
    """librosa.hz_to_mel(htk=False): the Slaney scale, linear below 1 kHz and logarithmic above."""
    frequencies = np.asanyarray(frequencies)
    f_min, f_sp = 0.0, 200.0 / 3
    mels = (frequencies - f_min) / f_sp
    min_log_hz = 1000.0
    min_log_mel = (min_log_hz - f_min) / f_sp
    logstep = np.log(6.4) / 27.0
    if frequencies.ndim:
        log_t = frequencies >= min_log_hz
        mels[log_t] = min_log_mel + np.log(frequencies[log_t] / min_log_hz) / logstep
    elif frequencies >= min_log_hz:
        mels = min_log_mel + np.log(frequencies / min_log_hz) / logstep
    return mels


def _mel_to_hz(mels):
    """librosa.mel_to_hz(htk=False)."""
    mels = np.asanyarray(mels)
    f_min, f_sp = 0.0, 200.0 / 3
    freqs = f_min + f_sp * mels
    min_log_hz = 1000.0
    min_log_mel = (min_log_hz - f_min) / f_sp
    logstep = np.log(6.4) / 27.0
    if mels.ndim:
        log_t = mels >= min_log_mel
        freqs[log_t] = min_log_hz * np.exp(logstep * (mels[log_t] - min_log_mel))
    elif mels >= min_log_mel:
        freqs = min_log_hz * np.exp(logstep * (mels - min_log_mel))
    return freqs


def mel_filterbank(sr, n_fft, n_mels=128, fmin=0.0, fmax=None):
    """librosa.filters.mel(sr=, n_fft=, n_mels=, fmin=, fmax=) with its defaults htk=False, norm="slaney", dtype=float32,
    restated with the same operations in the same order: (n_mels, 1 + n_fft // 2) float32."""
    if fmax is None:
        fmax = float(sr) / 2
    n_mels = int(n_mels)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)), dtype=np.float32)
    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


def band_table(basis):
    """Dense (n_mels, n_bins) float32 basis -> (bands (n_mels, 3) int32 {first bin, bin count, offset}, weights float32): each
    band's entries from its first to its last nonzero bin.  An all-zero band has count 0."""
    basis = np.asarray(basis, dtype=np.float32)
    bands = np.zeros((basis.shape[0], 3), np.int32)
    parts, off = [], 0
    for j, row in enumerate(basis):
        nz = np.nonzero(row)[0]
        first, cnt = (int(nz[0]), int(nz[-1]) - int(nz[0]) + 1) if nz.size else (0, 0)
        bands[j] = (first, cnt, off)
        parts.append(row[first:first + cnt])
        off += cnt
    return bands, (np.concatenate(parts) if off else np.zeros(1, np.float32)).astype(np.float32)


def hann_window_scipy():
    """fp32(scipy.signal.get_window('hann', 1024, fftbins=True)): the window of stft.py:121-123 and of librosa.stft."""
    from scipy.signal import get_window
    return get_window("hann", N_FFT, fftbins=True).astype(np.float32)


def twiddles():
    """(1024, 2) float32 (cos, -sin)(2 pi k / 1024), computed in fp64 and rounded."""
    a = 2.0 * np.pi * np.arange(N_FFT, dtype=np.float64) / N_FFT
    return np.stack([np.cos(a), -np.sin(a)], axis=1).astype(np.float32)


def n_frames(n, pad, hop):
    """Frames of an n-sample item reflect-padded by pad at both ends (conv1d / stft with center=False)."""
    return (int(n) + 2 * int(pad) - N_FFT) // int(hop) + 1


def _check_hop(hop):
    if not (1 <= int(hop) <= N_FFT):
        raise ValueError("hop length %d is not supported: it must be in [1, 1024]" % int(hop))


def _check_fft(n_fft, win_length):
    if int(n_fft) != N_FFT or int(win_length) != N_FFT:
        raise ValueError("n_fft %d / win_length %d are not supported: the FFT size is 1024 and the window spans all of it"
                         % (int(n_fft), int(win_length)))


def _lengths(y, lengths, pad):
    """Host item lengths (``recordings.host_lengths``), checked like F.pad(reflect) would."""
    ls = recordings.host_lengths(lengths, *y.shape)
    for v in ls:
        if v <= pad:
            raise RuntimeError("an item of %d samples is not longer than the reflect padding %d" % (v, pad))
        if v + 2 * pad < N_FFT:
            raise RuntimeError("an item of %d samples padded by %d on each side is shorter than the 1024-point frame" % (v, pad))
    return ls


def _checked_band_table(basis):
    bt, bw = band_table(basis)
    if bt.shape[0] > _MAX_MELS:
        raise ValueError("%d mel bands are not supported: at most %d" % (bt.shape[0], _MAX_MELS))
    return bt, bw


def device_bands(basis, dev):
    """band_table of a dense basis as device tensors (bands, weights)."""
    bt, bw = _checked_band_table(basis.detach().cpu().numpy() if torch.is_tensor(basis) else basis)
    return torch.from_numpy(bt).to(dev), torch.from_numpy(bw).to(dev)


def mel_bands(sampling_rate, num_mels, fmin, fmax, dev):
    """device_bands of mel_filterbank(sampling_rate, 1024, num_mels, fmin, fmax), made once per device like the reference's
    mel_basis dict."""
    key = ("mel_bands", int(sampling_rate), int(num_mels), float(fmin), None if fmax is None else float(fmax))
    return recordings.device_table(key, lambda: _checked_band_table(
        mel_filterbank(sr=sampling_rate, n_fft=N_FFT, n_mels=num_mels, fmin=fmin, fmax=fmax)), dev)


def scipy_hann(dev):
    """hann_window_scipy() on dev, made once per device."""
    return recordings.device_table("scipy_hann", hann_window_scipy, dev)


def stft_features(y, pad, hop, window, mag_eps, bands=None, energy=False, lengths=None, check_range=False):
    """One launch of the fused kernel on y (B, N): -> (mel (B, n_mels, F) or None, energy (B, F) or None, status word or None).
    bands: device_bands(basis) or None; F = n_frames(N, pad, hop); frames past an item's own count are 0."""
    _check(y, "y")
    _check_hop(hop)
    if y.dim() != 2:
        raise ValueError("expected a (B, N) waveform, got shape %s" % (tuple(y.shape),))
    ls = _lengths(y, lengths, pad)
    lib = _abi.load()
    dev = y.device
    x = y.detach().to(torch.float32).contiguous()
    B, N = x.shape
    F = n_frames(N, pad, hop)
    mel = out_e = band_w = None
    n_mels = 0
    if bands is not None:
        bands, band_w = bands
        n_mels = bands.shape[0]
        mel = torch.empty((B, n_mels, F), dtype=torch.float32, device=dev)
    if energy:
        out_e = torch.empty((B, F), dtype=torch.float32, device=dev)
    ns = None if lengths is None else recordings.upload([ls], dev)[0]
    status = torch.zeros(1, dtype=torch.int32, device=dev) if check_range else None
    win = window.detach().to(device=dev, dtype=torch.float32).contiguous()
    tw = recordings.device_table("twiddles", twiddles, dev)
    _abi.check(lib.ev_stft_features(x.data_ptr(), N, None if ns is None else ns.data_ptr(), B, int(pad), int(hop), F, win.data_ptr(),
                                    tw.data_ptr(), float(mag_eps), None if bands is None else bands.data_ptr(),
                                    None if band_w is None else band_w.data_ptr(), n_mels, None if mel is None else mel.data_ptr(),
                                    None if out_e is None else out_e.data_ptr(), None if status is None else status.data_ptr(),
                                    torch.cuda.current_stream(dev).cuda_stream))
    return mel, out_e, status


class TacotronSTFT(nn.Module):
    """tacotron_stft.py:46-80 with the reference's constructor.  ``mel_spectrogram(y)``: y (B, N) CUDA float in [-1, 1] ->
    (B, n_mel_channels, N // hop_length + 1) float32.  No inverse and no phases."""

    def __init__(self, filter_length=1024, hop_length=256, win_length=1024, n_mel_channels=80, sampling_rate=22050, mel_fmin=0.0,
                 mel_fmax=8000.0):
        super().__init__()
        _check_fft(filter_length, win_length)
        _check_hop(hop_length)
        self.n_mel_channels = n_mel_channels
        self.sampling_rate = sampling_rate
        self.filter_length, self.hop_length, self.win_length = int(filter_length), int(hop_length), int(win_length)
        mel_basis = mel_filterbank(sr=sampling_rate, n_fft=filter_length, n_mels=n_mel_channels, fmin=mel_fmin, fmax=mel_fmax)
        self.register_buffer("mel_basis", torch.from_numpy(mel_basis).float())
        self.register_buffer("window", torch.from_numpy(hann_window_scipy()))
        self._bands = None

    def mel_spectrogram(self, y, lengths=None):
        """Raises AssertionError, like the reference's asserts (tacotron_stft.py:73-74), when a sample of an item is outside
        [-1, 1]; reading the kernel's status word back is the call's one sync."""
        _check(y, "y")
        dev = y.device
        if self._bands is None or self._bands[0] != (dev, self.mel_basis._version):
            self._bands = ((dev, self.mel_basis._version), device_bands(self.mel_basis, dev))
        mel, _, status = stft_features(y, self.filter_length // 2, self.hop_length, self.window.to(dev), 0.0, bands=self._bands[1],
                                       lengths=lengths, check_range=True)
        if int(status.item()) & _STATUS_RANGE:
            raise AssertionError("TacotronSTFT.mel_spectrogram: a sample is outside [-1, 1]")
        return mel


def mel_spectrogram_torch(y, n_fft, num_mels, sampling_rate, hop_size, win_size, fmin, fmax, center=False, lengths=None):
    """mel_process.py:77-110: y (B, N) CUDA float -> (B, num_mels, F), F = (N + 2p - n_fft) // hop_size + 1 with
    p = (n_fft - hop_size) // 2.  Out-of-range samples are not checked (the reference only prints them)."""
    _check(y, "y")
    _check_fft(n_fft, win_size)
    _check_hop(hop_size)
    if center:
        raise ValueError("mel_spectrogram_torch: center=True is not supported, only the reference's center=False")
    dev = y.device
    bands = mel_bands(sampling_rate, num_mels, fmin, fmax, dev)
    window = recordings.device_table("torch_hann", lambda: torch.hann_window(N_FFT).numpy(), dev)
    mel, _, _ = stft_features(y, (N_FFT - int(hop_size)) // 2, hop_size, window, 1e-6, bands=bands, lengths=lengths)
    return mel


class Energy:
    """feats.py:159-213 with the reference's constructor.  ``get_energy(wav)``: wav (N,) or (B, N) CUDA float -> frame energy
    (F,) or (B, F), F = N // hop_length + 1; with ``duration`` (1-D input) the per-token means.  The caller keeps the
    ``energy_stats`` normalisation (prompt_dataset.py:141)."""

    def __init__(self, sr=24000, n_fft=2048, hop_length=300, win_length=None, window="hann", center=True, pad_mode="reflect"):
        self.sr = sr
        self.n_fft = n_fft
        self.win_length = win_length
        self.hop_length = hop_length
        self.window = window
        self.center = center
        self.pad_mode = pad_mode
        _check_fft(n_fft, n_fft if win_length is None else win_length)
        _check_hop(hop_length)
        if window != "hann":
            raise ValueError("window %r is not supported: only 'hann'" % (window,))
        if not center:
            raise ValueError("Energy(center=False) is not supported, only center=True")
        if pad_mode != "reflect":
            raise ValueError("pad_mode %r is not supported: only 'reflect'" % (pad_mode,))

    def _calculate_energy(self, wav, lengths=None):
        _, e, _ = stft_features(wav, N_FFT // 2, self.hop_length, scipy_hann(wav.device), 0.0, energy=True, lengths=lengths)
        return e

    def get_energy(self, wav, use_token_averaged_energy=True, duration=None, lengths=None):
        _check(wav, "wav")
        one = wav.dim() == 1
        average = use_token_averaged_energy and duration is not None
        if average and not one:
            raise ValueError("duration is per item: token averaging takes a 1-D waveform, as in the reference")
        energy = self._calculate_energy(wav[None] if one else wav, lengths)
        if average:
            return self._average_by_duration(energy, duration)[0]
        return energy[0] if one else energy

    def _average_by_duration(self, energy, d):
        """feats.py:198-207 through ev_op_average_by_duration: energy (1, F), d (T,) -> (1, T)."""
        from . import align
        d = (d.detach() if torch.is_tensor(d) else torch.from_numpy(np.asarray(d))).to(device=energy.device, dtype=torch.float32).reshape(1, -1)
        T, F = d.shape[1], energy.shape[1]
        return align.average_by_duration(d, energy, torch.tensor([T]), torch.tensor([F]))


# ---- pitch ---------------------------------------------------------------------------------------------------------------
PITCH_SR_RANGE = (8000, 48000)    # Hz, integers: covers 16, 22.05, 24 and 48 kHz
PITCH_HOP_RANGE = (16, 4096)      # samples
_PITCH_CONTINUOUS, _PITCH_LOG = 1, 2


def pitch_frame_period(sr, hop):
    """feats.py:119: the frame period in ms handed to pyworld.dio."""
    return 1000 * hop / sr


def pitch_frames(n, sr, hop):
    """pyworld's frame count of an n-sample item, int(1000 n / fs / frame_period) + 1 in double (N // hop + 1 at the configs)."""
    return int(1000.0 * int(n) / int(sr) / pitch_frame_period(sr, hop)) + 1


def pitch_min_samples(sr):
    """The shortest item get_pitch takes: the length of DIO's 50 Hz low-cut filter, 2 round(sr / 50) + 1 samples."""
    return 2 * int(sr / 50.0 + 0.5) + 1


def _check_pitch_config(sr, hop):
    if int(sr) != sr or not PITCH_SR_RANGE[0] <= int(sr) <= PITCH_SR_RANGE[1]:
        raise ValueError("sample rate %r is not supported: it must be an integer in [%d, %d] Hz" % ((sr,) + PITCH_SR_RANGE))
    if int(hop) != hop or not PITCH_HOP_RANGE[0] <= int(hop) <= PITCH_HOP_RANGE[1]:
        raise ValueError("hop length %r is not supported: it must be an integer in [%d, %d]" % ((hop,) + PITCH_HOP_RANGE))


def _pitch_input(wav, sr, hop, lengths):
    """The checks of pitch_track and spectral_envelope -> host lengths."""
    _check(wav, "wav")
    _check_pitch_config(sr, hop)
    if wav.dim() != 2:
        raise ValueError("expected a (B, N) waveform, got shape %s" % (tuple(wav.shape),))
    if wav.dtype not in (torch.float32, torch.float64):
        raise ValueError("wav must be float32 or float64, got %s" % wav.dtype)
    B, N = wav.shape
    ls = recordings.host_lengths(lengths, B, N)
    m = pitch_min_samples(sr)
    if any(v < m for v in ls):
        raise ValueError("an item of %d samples is too short to filter: at least %d at %d Hz" % (min(ls), m, int(sr)))
    return ls


def pitch_track(wav, sr, hop, continuous=True, log=False, lengths=None, raw=False):
    """One ev_pitch call on wav (B, N) CUDA float32/float64 -> pitch (B, F) float64 [, DIO's raw contour (B, F)],
    F = pitch_frames(N, sr, hop); frames past an item's own count are 0."""
    ls = _pitch_input(wav, sr, hop, lengths)
    B, N = wav.shape
    lib = _abi.load()
    dev = wav.device
    x = wav.detach().to(torch.float64).contiguous()
    fp = pitch_frame_period(int(sr), int(hop))
    F = pitch_frames(N, sr, hop)
    nbytes = lib.ev_pitch_workspace_bytes(B, N, int(sr), fp, F)
    if nbytes == 0:
        raise ValueError("ev_pitch rejects B=%d N=%d sr=%d hop=%d" % (B, N, int(sr), int(hop)))
    ws = torch.empty((nbytes + 15) // 16 * 2, dtype=torch.float64, device=dev)
    ns = None if lengths is None else recordings.upload([ls], dev)[0]
    out = torch.empty((B, F), dtype=torch.float64, device=dev)
    f0 = torch.empty((B, F), dtype=torch.float64, device=dev) if raw else None
    flags = (_PITCH_CONTINUOUS if continuous else 0) | (_PITCH_LOG if log else 0)
    _abi.check(lib.ev_pitch(x.data_ptr(), N, None if ns is None else ns.data_ptr(), B, int(sr), fp, F, flags,
                            None if f0 is None else f0.data_ptr(), out.data_ptr(), None, ws.data_ptr(), ws.numel() * 8,
                            torch.cuda.current_stream(dev).cuda_stream))
    return (out, f0) if raw else out


class Pitch:
    """feats.py:83-156 with the reference's constructor.  ``get_pitch(wav)``: wav (N,) or (B, N) CUDA float32/float64 -> F0 in Hz
    (F,) or (B, F) float64, F = pyworld's frame count (N // hop_length + 1 at 16 kHz / 256 and 24 kHz / 300): pyworld.dio and
    pyworld.stonemask at their defaults (restated; not checked against pyworld), then optionally the continuous interpolation
    and the log.  With ``use_token_averaged_pitch`` and ``duration`` (1-D input) the per-token means, through
    ``align.average_by_duration`` (fp32).  ``pitch_min`` / ``pitch_max`` are kept and unused, as in the reference, which never
    passes them to dio.  The caller keeps the ``pitch_stats`` normalisation (prompt_dataset.py:140)."""

    def __init__(self, sr=24000, hop_length=300, pitch_min=80, pitch_max=7600):
        self.sr = sr
        self.hop_length = hop_length
        self.pitch_min = pitch_min
        self.pitch_max = pitch_max
        _check_pitch_config(sr, hop_length)

    def get_pitch(self, wav, use_continuous_pitch=True, use_log_pitch=False, use_token_averaged_pitch=False, duration=None,
                  lengths=None):
        _check(wav, "wav")
        one = wav.dim() == 1
        average = use_token_averaged_pitch and duration is not None
        if average and not one:
            raise ValueError("duration is per item: token averaging takes a 1-D waveform, as in the reference")
        p = pitch_track(wav[None] if one else wav, self.sr, self.hop_length, use_continuous_pitch, use_log_pitch, lengths)
        if average:
            return self._average_by_duration(p, duration)[0].to(torch.float64)
        return p[0] if one else p

    def _average_by_duration(self, pitch, d):
        """feats.py:133-147 (its zero mask is a no-op) through ev_op_average_by_duration: pitch (1, F), d (T,) -> (1, T) float32."""
        from . import align
        d = (d.detach() if torch.is_tensor(d) else torch.from_numpy(np.asarray(d))).to(device=pitch.device, dtype=torch.float32).reshape(1, -1)
        T, F = d.shape[1], pitch.shape[1]
        return align.average_by_duration(d, pitch, torch.tensor([T]), torch.tensor([F]))


# ---- spectral envelope and mel-cepstrum -------------------------------------------------------------------------------------
SP2MC_MAX_ORDER = 255


def world_fft_size(sr):
    """pyworld.cheaptrick's default FFT size at sr Hz: 2^(1 + int(log(3 sr / 71 + 1) / log 2)) (512 at 8 kHz, 1024 at 16 to
    24 kHz, 2048 at 44.1 and 48 kHz)."""
    return 2 ** (1 + int(np.log(3.0 * sr / 71.0 + 1.0) / np.log(2.0)))


def sp2mc_table(n_fft, order, alpha):
    """(order + 1, n_fft // 2 + 1) float64: the matrix of pysptk.sp2mc(sp, order, alpha) on log(sp), i.e. c = irfft(log sp),
    c[0] /= 2, then SPTK's freqt(c, order, alpha) over all n_fft coefficients of c, its mirror half included.  Built by running
    the freqt recursion on the columns of the irfft matrix in fp64."""
    bins = n_fft // 2 + 1
    c = np.fft.irfft(np.eye(bins), n=n_fft, axis=1).T          # (n_fft, bins): c = c_of_log @ log sp
    c[0] /= 2.0
    a, b = float(alpha), 1.0 - float(alpha) * float(alpha)
    g = np.zeros((order + 1, bins))
    for i in range(n_fft - 1, -1, -1):
        d = g.copy()
        g[0] = c[i] + a * d[0]
        if order >= 1:
            g[1] = b * d[0] + a * d[1]
        for j in range(2, order + 1):
            g[j] = d[j - 1] + a * (d[j] - g[j - 1])
    return g


def _check_sp2mc(order, alpha):
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or not 0 <= int(order) <= SP2MC_MAX_ORDER:
        raise ValueError("order must be an integer in [0, %d], got %r" % (SP2MC_MAX_ORDER, order))
    if isinstance(alpha, bool) or not isinstance(alpha, (int, float, np.integer, np.floating)) or not abs(float(alpha)) < 1.0:
        raise ValueError("alpha must be a number with |alpha| < 1, got %r" % (alpha,))


def mcep_table(n_fft, order, alpha, dev, first=0):
    """Rows first..order of sp2mc_table(n_fft, order, alpha) on dev, made once per device."""
    key = ("sp2mc", int(n_fft), int(order), float(alpha), int(first))
    return recordings.device_table(key, lambda: np.ascontiguousarray(sp2mc_table(int(n_fft), int(order), float(alpha))[first:]), dev)


def envelope_features(wav, sr, hop, f0=None, lengths=None, table=None, envelope=True):
    """One ev_world_envelope call -> (sp (B, F, bins) float64 or None, table @ log sp (B, F, rows) float64 or None).  The
    arguments are spectral_envelope's; table: a device (rows, bins) float64 table or None."""
    ls = _pitch_input(wav, sr, hop, lengths)
    B, N = wav.shape
    F = pitch_frames(N, sr, hop)
    if f0 is None:
        f0 = pitch_track(wav, sr, hop, continuous=False, lengths=lengths)
    elif not (torch.is_tensor(f0) and f0.device == wav.device and f0.dtype == torch.float64 and tuple(f0.shape) == (B, F)):
        raise ValueError("f0 must be a (%d, %d) float64 tensor on %s" % (B, F, wav.device))
    lib = _abi.load()
    dev = wav.device
    x = wav.detach().to(torch.float64).contiguous()
    f0 = f0.detach().contiguous()
    bins = world_fft_size(int(sr)) // 2 + 1
    sp = torch.empty((B, F, bins), dtype=torch.float64, device=dev) if envelope else None
    mc = None if table is None else torch.empty((B, F, int(table.shape[0])), dtype=torch.float64, device=dev)
    ns = None if lengths is None else recordings.upload([ls], dev)[0]
    _abi.check(lib.ev_world_envelope(x.data_ptr(), N, None if ns is None else ns.data_ptr(), B, int(sr),
                                     pitch_frame_period(int(sr), int(hop)), F, f0.data_ptr(), None if sp is None else sp.data_ptr(),
                                     None if table is None else table.data_ptr(), 0 if table is None else int(table.shape[0]),
                                     None if mc is None else mc.data_ptr(), None, torch.cuda.current_stream(dev).cuda_stream))
    return sp, mc


def spectral_envelope(wav, sample_rate, hop, f0=None, lengths=None):
    """pyworld.cheaptrick at its defaults (q1 = -0.15, f0_floor 71, fft_size = world_fft_size(sample_rate)) on the GPU in fp64
    (``ev_world_envelope``; oracle/world_oracle.py lists every assumed detail, not checked against pyworld).

    wav (B, N) CUDA float32/float64 at ``sample_rate`` Hz with the frames of ``pitch_track(wav, sample_rate, hop)`` (frame
    period 1000 hop / sample_rate ms); ``f0``: their F0, a (B, F) float64 tensor on wav's device, or None for
    ``pitch_track(continuous=False)``; ``lengths`` as pitch_track's.  Returns the power envelope (B, F, fft_size // 2 + 1)
    float64; frames past an item's own count are 0.  WORLD's random noise is replaced by a floor of 2^-52 on every power
    bin, so each item's envelope is the same in any batch and silence gives finite values.  No host sync."""
    return envelope_features(wav, sample_rate, hop, f0, lengths)[0]


def sp2mc(sp, order, alpha):
    """pysptk.sp2mc(sp, order, alpha) on the GPU (``ev_sp2mc``): sp a CUDA float64 (..., bins) power envelope, bins =
    fft_size // 2 + 1 with fft_size a power of two in [4, 2048], every value > 0 -> (..., order + 1) float64 mel-cepstra.
    order in [0, 255], |alpha| < 1.  The map is ``sp2mc_table`` (fp64, built once per (fft_size, order, alpha) and device)
    applied to log(sp)."""
    _check_sp2mc(order, alpha)
    if not (torch.is_tensor(sp) and sp.is_cuda and sp.dtype == torch.float64 and sp.dim() >= 1):
        raise ValueError("sp must be a CUDA float64 tensor (..., bins)")
    bins = int(sp.shape[-1])
    n_fft = 2 * (bins - 1)
    if bins < 3 or n_fft > 2048 or n_fft & (n_fft - 1):
        raise ValueError("sp has %d bins: it must have fft_size // 2 + 1 with fft_size a power of two in [4, 2048]" % bins)
    lib = _abi.load()
    dev = sp.device
    x = sp.detach().contiguous()
    table = mcep_table(n_fft, int(order), float(alpha), dev)
    out = torch.empty(tuple(sp.shape[:-1]) + (int(order) + 1,), dtype=torch.float64, device=dev)
    _abi.check(lib.ev_sp2mc(x.data_ptr(), x.numel() // bins, bins, table.data_ptr(), int(order) + 1, out.data_ptr(),
                            torch.cuda.current_stream(dev).cuda_stream))
    return out
