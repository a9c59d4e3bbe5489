"""CPU: capture files into ``Signal`` (reference: src/urh/signalprocessing/Signal.py:114-213, IQArray.py:206-227) - wav (8 / 16 / 24 /
32 bit, one and two channels), Flipper ``.sub`` run lengths, ``.coco`` archives and the raw sample formats by file extension -
loaded by urh_b200.signalprocessing.Signal and by the reference's own class: same samples, dtype, sample rate and
already-demodulated flag.  The noise threshold is fixed through the settings so that no GPU is needed (with "automatic" the
constructor runs detect_noise_level on the device).  The reference's answers are recorded in tests/golden/ref_signal_files.json
(oracle/cassette.py)."""
import tarfile
import wave

import numpy as np
import pytest

from oracle.cassette import RECORD, Cassette, same


@pytest.fixture
def cassette(request):
    c = Cassette("signal_files", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def classes():
    from urh_b200 import settings
    from urh_b200.signalprocessing.Signal import Signal

    ref_cls = None
    if RECORD:
        from oracle import ref_loader
        ref_cls = ref_loader.load_python_layer().Signal
    settings.write("default_noise_threshold", "3")
    yield Signal, ref_cls
    settings.write("default_noise_threshold", "automatic")


def both(cassette, classes, path):
    mine_cls, ref_cls = classes
    mine, ref = mine_cls(str(path), "t"), cassette.make(lambda: ref_cls(str(path), "t"))
    a = np.asarray(mine.iq_array.data)
    assert a.dtype == cassette.want(lambda: np.asarray(ref.iq_array.data).dtype)
    assert a.shape == cassette.want(lambda: np.asarray(ref.iq_array.data).shape)
    assert same(a.view(np.uint8), cassette.want(lambda: np.asarray(ref.iq_array.data).view(np.uint8)))   # bit-identical samples
    assert mine.sample_rate == cassette.want(lambda: ref.sample_rate)
    assert mine.already_demodulated == cassette.want(lambda: ref.already_demodulated)
    assert mine.wav_mode == cassette.want(lambda: ref.wav_mode)
    assert mine.num_samples == cassette.want(lambda: ref.num_samples)
    return mine


@pytest.mark.parametrize("width", [1, 2, 3, 4])
@pytest.mark.parametrize("channels", [1, 2])
def test_wav(cassette, classes, tmp_path, width, channels):
    rng = np.random.default_rng(10 * width + channels)
    frames, rate = 1234, 48000 if channels == 1 else 250000
    raw = rng.integers(0, 256, frames * channels * width, dtype=np.uint8).tobytes()
    path = tmp_path / ("c%d_w%d.wav" % (channels, width))
    with wave.open(str(path), "w") as f:
        f.setnchannels(channels)
        f.setsampwidth(width)
        f.setframerate(rate)
        f.writeframes(raw)
    mine = both(cassette, classes, path)
    assert mine.sample_rate == rate
    assert mine.already_demodulated == (channels == 1)


def test_flipper_sub(cassette, classes, tmp_path):
    path = tmp_path / "remote.sub"
    path.write_text("Filetype: Flipper SubGhz RAW File\nVersion: 1\nFrequency: 433920000\nProtocol: RAW\n"
                    "RAW_Data: 300 -900 300 -300 900 -9000\nRAW_Data: 450 -450 1350 -100\nsomething else: 5\n")
    mine = both(cassette, classes, path)
    assert mine.already_demodulated and mine.num_samples == 300 + 900 + 300 + 300 + 900 + 9000 + 450 + 450 + 1350 + 100


@pytest.mark.parametrize("ext,dtype", [(".complex", np.float32), (".cs8", np.int8), (".complex16s", np.int8), (".cs16", np.int16),
                                       (".complex32s", np.int16)])
def test_raw_formats_and_coco(cassette, classes, tmp_path, ext, dtype):
    rng = np.random.default_rng(len(ext))
    n = 777
    if dtype == np.float32:
        data = rng.standard_normal((n, 2)).astype(np.float32)
    else:
        info = np.iinfo(dtype)
        data = rng.integers(info.min, info.max + 1, (n, 2)).astype(dtype)
    path = tmp_path / ("capture" + ext)
    data.tofile(str(path))
    mine = both(cassette, classes, path)
    assert mine.iq_array.data.dtype == dtype and np.array_equal(mine.iq_array.data, data)
    # the same file inside a .coco archive (Signal.py:190-205)
    coco = tmp_path / ("capture" + ext.replace(".", "_") + ".coco")
    with tarfile.open(str(coco), "w:bz2") as tar:
        tar.add(str(path), arcname="capture" + ext)
    mine2 = both(cassette, classes, coco)
    assert np.array_equal(mine2.iq_array.data, data)


@pytest.mark.gpu
@pytest.mark.parametrize("ext,dtype", [(".cu8", np.uint8), (".complex16u", np.uint8), (".cu16", np.uint16), (".complex32u", np.uint16)])
def test_unsigned_formats_become_signed(tmp_path, ext, dtype):
    """unsigned captures are handled as signed (IQArray.py:214-218): the conversion runs on the device (convert.cu)"""
    from urh_b200 import settings
    from urh_b200.signalprocessing.Signal import Signal

    info = np.iinfo(dtype)
    data = np.random.default_rng(len(ext)).integers(info.min, info.max + 1, (999, 2)).astype(dtype)
    data[0], data[1] = info.min, info.max
    path = tmp_path / ("capture" + ext)
    data.tofile(str(path))
    settings.write("default_noise_threshold", "3")
    try:
        sig = Signal(str(path), "t")
    finally:
        settings.write("default_noise_threshold", "automatic")
    signed = np.int8 if dtype == np.uint8 else np.int16
    half = 128 if dtype == np.uint8 else 32768
    assert sig.iq_array.data.dtype == signed
    assert np.array_equal(sig.iq_array.data, (data.astype(np.int64) - half).astype(signed))
