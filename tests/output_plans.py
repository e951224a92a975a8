"""The plans the output chain runs for every output rate ``audio.plan`` accepts from the model's 16 kHz, and the representative
rates tests/test_output_kernels_gpu.py checks the chain's kernels at.

Each accepted rate is classified by what changes the kernels' code paths or launch shapes:

* ev_format_audio's resampler: the copy, up > down or down > up, with the taps per phase, the input window of a 256-output
  tile and the dynamic shared memory that ``launch_audio_out`` computes from up and down;
* ev_limit's detector bank from ``audio.limit_bank``: phases, taps and hold M;
* ev_flac_encode's frame-header sample-rate code: one of the eleven standard codes, 12 (8-bit kHz), 13 (16-bit Hz), 14 (16-bit
  tens of Hz) or 0 (the rate only in STREAMINFO);
* whether a watermark may be asked for (8000 Hz and above).

``CLASSES`` names the sets of rates that must each hold a representative: every kind of the four classifications, and every
rate at an extreme (lowest and highest rate, largest up and down, most taps per phase, widest window, most shared memory,
widest and narrowest low-passed limiter bank, largest hold, the watermark's lowest rate).
"""
import functools

from emotivoice_b200 import audio

SOURCE_RATE = 16000
AO_TILE = 256                   # outputs per audio_out_kernel tile (voc_kernels.cu)

# rate: why it is here
REPRESENTATIVE_RATES = {
    4000: "1/4: lowest rate, most taps per phase (81) and widest window; FLAC code 12; limiter bank 12 x 101, M = 50",
    4016: "251/1000: largest down; FLAC code 13; limiter bank 12 x 101",
    8000: "1/2: standard FLAC code; the watermark's lowest rate",
    11025: "441/640: FLAC code 13",
    12000: "3/4: FLAC code 12",
    15625: "125/128: just below the source rate; FLAC code 13; narrowest low-passed limiter bank, 12 x 43",
    16000: "the copy; standard FLAC code",
    16368: "1023/1000: most shared memory (87,016 B)",
    65600: "41/10: FLAC code 14",
    127625: "1021/128: FLAC code 0",
    131072: "1024/125: largest up; FLAC code 0",
    192000: "12/1: highest rate; standard FLAC code 3",
}


def resampler(up, down):
    """ev_format_audio's plan for up / down -> (kind, taps per phase, window, dynamic shared memory bytes), as
    ``launch_audio_out`` computes them."""
    if up == down == 1:
        return "copy", 0, 0, 0
    half = 10 * max(up, down)
    taps = (2 * half + 1 + up - 1) // up
    window = ((AO_TILE - 1) * down + up - 1) // up + taps
    return ("up" if up > down else "down"), taps, window, (up * taps + window) * 4


@functools.lru_cache(maxsize=None)
def plans():
    """rate -> dict of its plan, for every rate ``audio.plan`` accepts from 16 kHz."""
    out = {}
    for rate in range(audio.RATE_RANGE[0], audio.RATE_RANGE[1] + 1):
        try:
            _, up, down = audio.plan(rate, "pcm16", SOURCE_RATE)
        except ValueError:
            continue
        kind, taps, window, smem = resampler(up, down)
        bank, hold = audio.limit_bank(SOURCE_RATE, rate)
        code = audio.flac_rate_code(rate)[0]
        out[rate] = dict(up=up, down=down, kind=kind, taps=taps, window=window, smem=smem, bank=bank.shape, hold=hold,
                         flac=code, flac_kind="standard" if code in audio.FLAC_STANDARD_RATES.values() else "code %d" % code,
                         watermark=rate >= audio.WATERMARK_MIN_RATE)
    return out


def _argmax(p, key, among=None):
    rates = [r for r in p if among is None or among(p[r])]
    best = max(key(p[r]) for r in rates)
    return {r for r in rates if key(p[r]) == best}


def classes():
    """name -> the set of accepted rates in that class; each must hold a representative rate."""
    p = plans()
    c = {}
    for kind in ("copy", "up", "down"):
        c["resampler %s" % kind] = {r for r in p if p[r]["kind"] == kind}
    c["limiter interpolator bank (phases 1 .. R - 1)"] = {r for r in p if p[r]["bank"][0] == 11}
    c["limiter low-passed bank (all R phases)"] = {r for r in p if p[r]["bank"][0] == 12}
    for kind in sorted({p[r]["flac_kind"] for r in p}):
        c["FLAC rate %s" % kind] = {r for r in p if p[r]["flac_kind"] == kind}
    c["watermark allowed"] = {r for r in p if p[r]["watermark"]}
    c["watermark refused"] = {r for r in p if not p[r]["watermark"]}
    lowpassed = lambda q: q["bank"][0] == 12
    c["lowest rate"] = {min(p)}
    c["highest rate"] = {max(p)}
    c["largest up"] = _argmax(p, lambda q: q["up"])
    c["largest down"] = _argmax(p, lambda q: q["down"])
    c["most taps per phase"] = _argmax(p, lambda q: q["taps"])
    c["widest window"] = _argmax(p, lambda q: q["window"])
    c["most shared memory"] = _argmax(p, lambda q: q["smem"])
    c["widest low-passed limiter bank"] = _argmax(p, lambda q: q["bank"][1], lowpassed)
    c["narrowest low-passed limiter bank"] = _argmax(p, lambda q: -q["bank"][1], lowpassed)
    c["largest limiter hold"] = _argmax(p, lambda q: q["hold"])
    c["watermark's lowest rate"] = {min(r for r in p if p[r]["watermark"])}
    return c


def uncovered(rates):
    """The names of the classes that none of ``rates`` falls in."""
    rates = set(rates)
    return sorted(name for name, members in classes().items() if not members & rates)
