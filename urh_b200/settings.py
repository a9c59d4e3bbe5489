"""Minimal stand-in for ``urh.settings`` (QSettings) — only the keys the IQ hot path reads
(reference: settings.py:157 read(), Signal.py:97, Modulator.py:68, Filter.py:50-56)."""
import os

_DEFAULTS = {
    "default_noise_threshold": "automatic",
    "modulation_dtype": "float32",
    "bandpass_filter_bw_type": "Medium",
    "bandpass_filter_custom_bw": 0.1,
}
_store = {}

CONTINUOUS_BUFFER_SIZE_MB = 50  # settings.py:38
SPECTRUM_BUFFER_SIZE = 2 ** 15  # settings.py:36
PIXELS_PER_PATH = 5000  # settings.py:35; path_creator.create_path reads it at call time


def read(key: str, default=None, type=None):
    env = os.environ.get("URH_" + key.upper())
    value = _store.get(key, env if env is not None else (_DEFAULTS.get(key) if default is None else default))
    if type is not None and value is not None:
        try:
            return type(value)
        except (TypeError, ValueError):
            return default
    return value


def write(key: str, value):
    _store[key] = value
