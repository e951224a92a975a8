"""The host side shared by every API that takes a batch of recordings (``emotivoice_b200.recordings``): ``host_lengths`` on
every input form, each entry point refusing non-integer lengths before the library is touched, and ``device_table``'s
cache; on the GPU, the cached tables and that ``meter``, ``detect`` and ``compare`` do not wait for the device once their
tables exist."""
import numpy as np
import pytest
import torch

from emotivoice_b200 import _abi, audio, evaluate, feats, loudness, recordings, watermark

B, L = 3, 1000


class _FakeCuda(torch.Tensor):
    """A CPU tensor that claims to be on the GPU, so the checks after the device check run without one."""
    @property
    def is_cuda(self):
        return True


class _FakeCudaLengths(torch.Tensor):
    """Integer lengths that claim to live on the GPU."""
    @property
    def device(self):
        return torch.device("cuda:0")


@pytest.mark.parametrize("lengths, want", [
    (None, [L] * B),
    ([0, 5, L], [0, 5, L]),
    ((0, 5, L), [0, 5, L]),
    (range(3), [0, 1, 2]),
    ([np.int32(7), np.int64(8), np.uint16(9)], [7, 8, 9]),
    (np.array([1, 2, 3], np.int64), [1, 2, 3]),
    (torch.tensor([4, 5, 6]), [4, 5, 6]),
    (torch.tensor([4, 5, 6], dtype=torch.int32), [4, 5, 6]),
])
def test_host_lengths_accepts_host_integers(lengths, want):
    got = recordings.host_lengths(lengths, B, L)
    assert got == want and all(type(v) is int for v in got)


@pytest.mark.parametrize("lengths, match", [
    ([1.5, 2, 3], "host integers"),
    ([2.0, 2, 3], "host integers"),
    ([True, 2, 3], "host integers"),
    ([np.bool_(True), 2, 3], "host integers"),
    (np.array([1.0, 2.0, 3.0]), "host integers"),
    (np.array([True, False, True]), "host integers"),
    (np.array(3), "host integers"),
    (torch.tensor([1.5, 2.0, 3.0]), "host integers"),
    (torch.tensor([True, False, True]), "host integers"),
    (torch.tensor(3), "host integers"),
    (torch.tensor([[1, 2, 3]]), "host integers"),
    (torch.tensor([1, 2, 3], device="meta"), "host integers"),
    (torch.tensor([1, 2, 3]).as_subclass(_FakeCudaLengths), "host integers"),
    ("123", "host integers"),
    (b"123", "host integers"),
    (["1", 2, 3], "host integers"),
    (3, "host integers"),
    ({1: 1, 2: 2, 3: 3}, "host integers"),
    ([1, 2], "2 lengths for 3 items"),
    ([1, 2, 3, 4], "4 lengths for 3 items"),
    ([-1, 2, 3], "-1 is negative"),
    ([1, 2, L + 1], "exceeds"),
])
def test_host_lengths_rejects_everything_else(lengths, match):
    with pytest.raises(ValueError, match=match):
        recordings.host_lengths(lengths, B, L)


def _no_library():
    raise AssertionError("the library was reached")


def _fake(b, n):
    return torch.zeros((b, n), dtype=torch.float32).as_subclass(_FakeCuda)


ENTRY_POINTS = {
    "stft_features": lambda ls: feats.stft_features(torch.zeros(2, 4000), 512, 256, torch.zeros(1024), 0.0, energy=True, lengths=ls),
    "TacotronSTFT": lambda ls: feats.TacotronSTFT(sampling_rate=16000).mel_spectrogram(torch.zeros(2, 4000), lengths=ls),
    "mel_spectrogram_torch": lambda ls: feats.mel_spectrogram_torch(torch.zeros(2, 4000), 1024, 80, 16000, 256, 1024, 0, 8000,
                                                                    lengths=ls),
    "Energy": lambda ls: feats.Energy(sr=16000, n_fft=1024, hop_length=256).get_energy(torch.zeros(2, 4000), lengths=ls),
    "pitch_track": lambda ls: feats.pitch_track(torch.zeros(2, 4000), 16000, 256, lengths=ls),
    "Pitch": lambda ls: feats.Pitch(sr=16000, hop_length=256).get_pitch(torch.zeros(2, 4000), lengths=ls),
    "meter": lambda ls: loudness.meter(_fake(2, 4000), 16000, lengths=ls),
    "detect": lambda ls: watermark.detect(_fake(2, 4000), 16000, 7, lengths=ls),
    "detect_48k": lambda ls: watermark.detect(_fake(2, 4000), 48000, 7, lengths=ls),
    "compare_syn": lambda ls: evaluate.compare(_fake(2, 4000), _fake(2, 4000), syn_lengths=ls),
    "compare_ref": lambda ls: evaluate.compare(_fake(2, 4000), _fake(2, 4000), ref_lengths=ls),
}


@pytest.mark.parametrize("name", sorted(ENTRY_POINTS))
@pytest.mark.parametrize("lengths", [[1.5, 4000], [True, 4000], [4000.0, 4000]])
def test_every_entry_point_refuses_non_integer_lengths_before_the_library(monkeypatch, name, lengths):
    monkeypatch.setattr(feats, "_check", lambda t, name: None)       # the feats APIs take these CPU tensors past their CUDA check
    monkeypatch.setattr(_abi, "load", _no_library)
    with pytest.raises(ValueError, match="host integers"):
        ENTRY_POINTS[name](lengths)


def test_device_table_makes_each_table_once_per_key_and_device(monkeypatch):
    monkeypatch.setattr(recordings, "_TABLES", {})
    calls = []

    def make(tag, value):
        def f():
            calls.append(tag)
            return value
        return f

    a = recordings.device_table("a", make("a", np.arange(4, dtype=np.float32)), "cpu")
    assert torch.is_tensor(a) and a.dtype == torch.float32 and a.tolist() == [0.0, 1.0, 2.0, 3.0]
    assert recordings.device_table("a", make("a again", None), "cpu") is a
    assert recordings.device_table("a", make("a again", None), torch.device("cpu")) is a
    pair = recordings.device_table(("b", 2), make("b", (np.ones(3, np.int32), 7)), "cpu")
    assert pair[0].dtype == torch.int32 and pair[0].tolist() == [1, 1, 1] and pair[1] == 7
    assert recordings.device_table(("b", 2), make("b again", None), "cpu") is pair
    assert recordings.device_table("none", make("none", None), "cpu") is None
    assert recordings.device_table("none", make("none again", np.zeros(1)), "cpu") is None
    assert calls == ["a", "b", "none"]


def test_k_weighting_is_one_host_table_per_rate():
    kc = loudness.k_weighting(48000)
    assert kc.device.type == "cpu" and kc.dtype == torch.float64 and kc.is_contiguous()
    assert np.array_equal(kc.numpy(), audio.k_weighting(48000))
    assert loudness.k_weighting(48000) is kc


@pytest.mark.gpu
def test_tables_uploads_and_batches_on_the_gpu():
    dev = torch.device("cuda:0")
    t = recordings.device_table("test_table", lambda: np.arange(5, dtype=np.float64), dev)
    assert t.device == dev and recordings.device_table("test_table", lambda: None, dev) is t
    assert recordings.device_table("test_table", lambda: np.zeros(5), "cuda:0") is t
    assert t.cpu().tolist() == [0.0, 1.0, 2.0, 3.0, 4.0]
    meta, (p_a, p_b) = recordings.upload([[1, 2, 3], np.array([4, 5], np.int64)], dev, np.int32)
    assert meta.dtype == torch.int32 and meta.cpu().tolist() == [1, 2, 3, 4, 5] and p_b == p_a + 12 == meta.data_ptr() + 12
    with pytest.raises(ValueError, match="host integers"):
        recordings.host_lengths(torch.tensor([1, 2, 3], device=dev), B, L)
    x = torch.zeros((4, 3000), device=dev)
    rows = x[:, :1000]                                # rows further apart than L: read in place
    assert recordings.recording_batch(rows).data_ptr() == rows.data_ptr()
    cols = torch.zeros((1000, 4), device=dev).t()     # samples not contiguous: copied
    got = recordings.recording_batch(cols)
    assert got.stride(1) == 1 and torch.equal(got, cols)
    wide = torch.zeros((1, 1000), device=dev).expand(4, 1000)          # overlapping rows: copied
    assert recordings.recording_batch(wide).stride(0) == 1000


@pytest.mark.gpu
def test_meter_detect_and_compare_do_not_wait_for_the_device():
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(5)
    w16 = 0.1 * torch.randn((2, 32000), device=dev, generator=g)
    w48 = 0.1 * torch.randn((2, 48000), device=dev, generator=g)
    r16 = w16.flip(0)
    calls = (lambda: loudness.meter(w16, 16000, lengths=[32000, 20000], series=True),
             lambda: loudness.meter(w48, 48000),
             lambda: watermark.detect(w16, 16000, 12345, lengths=[32000, 20000]),
             lambda: watermark.detect(w48, 48000, 12345, lengths=[48000, 30000]),
             lambda: evaluate.compare(w16, r16, syn_lengths=[32000, 20000], return_path=True))
    for f in calls:                               # the first call on a device builds its tables
        f()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for f in calls:
            f()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
