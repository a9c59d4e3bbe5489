"""Vectorised numpy restatement of the reference's FTA record assembly (Spectrogram.export_to_fta, Spectrogram.py:118-154), the
oracle the device export is compared with byte for byte.  The reference fills the record array in a Python double loop, one
structured element per (frequency bin, frame) cell; here the same values are broadcast at once."""
import numpy as np


def fta_dtype(include_amplitude):
    if include_amplitude:
        return np.dtype([("f", np.float64), ("t", np.uint32), ("a", np.float32)])
    return np.dtype([("f", np.float64), ("t", np.uint32)])


def fta_bytes(db, n, sample_rate, include_amplitude=False):
    """the bytes export_to_fta writes for the fliplr'ed dB map ``db`` [frames][W] of a capture of ``n`` samples.  Raises what the
    reference's loop raises at its first record whose time does not fit a uint32."""
    spectrogram = np.flipud(np.asarray(db, dtype=np.float32).T)   # [W][frames]
    W, F = spectrogram.shape
    dtype = fta_dtype(include_amplitude)
    fft_freqs = np.fft.fftshift(np.fft.fftfreq(W, 1 / sample_rate))
    time_width = 1e9 * ((n / sample_rate) / F)
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.arange(F, dtype=np.float64) * time_width   # j * time_width: j is exact in a double
        bad = ~np.isfinite(p) | (p >= 4294967296.0) | (p <= -1.0)
    if bad.any():
        j = int(np.argmax(bad))
        rec = np.empty(1, dtype=dtype)
        rec[0] = (fft_freqs[0], int(j * time_width)) + ((spectrogram[0, j],) if include_amplitude else ())
        raise AssertionError("the record above must raise")
    k = 3 if include_amplitude else 2
    result = np.empty((W, F, k), dtype=dtype)
    result["f"] = fft_freqs[:, None, None]
    result["t"] = np.trunc(p).astype(np.uint32)[None, :, None]
    if include_amplitude:
        result["a"] = spectrogram[:, :, None]
    return result.tobytes()
