"""tests/golden/g711.npz: G.711 of every int16 value, as Python's audioop computes it for 16-bit samples.

    python oracle/make_golden_g711.py

ulaw[i] = audioop.lin2ulaw(int16 i - 32768), alaw[i] likewise with lin2alaw (uint8, 65,536 entries each).  audioop is
deprecated and gone from Python 3.13, so the tables are kept as a fixture and the tests never import it.
"""
import os
import warnings

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "g711.npz")


def main():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        import audioop
    pcm = np.arange(-32768, 32768, dtype=np.int64).astype("<i2").tobytes()
    ulaw = np.frombuffer(audioop.lin2ulaw(pcm, 2), dtype=np.uint8)
    alaw = np.frombuffer(audioop.lin2alaw(pcm, 2), dtype=np.uint8)
    assert ulaw.shape == alaw.shape == (65536,)
    np.savez_compressed(OUT, ulaw=ulaw, alaw=alaw)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
