"""A plain numpy / Python restatement of IQArray.export_to_sub (IQArray.py:275-319): the entries the reference's sample loop appends
and the file it writes.  Pinned to the reference's own files in tests/test_sub_export_cpu.py; the device export is compared with it in
tests/test_gpu_sub_export.py.

The loop keeps (lastvalue, counter).  Restated as a chain of armed positions p (lastvalue = u[p], counter = 1):

    q = first index > p with u[q] == u[p]     (the samples in between are skipped: counted nowhere)
    no such q:  emit(1, u[p]) and stop
    r = end of the run of u[p] that starts at q
    emit(1 + r - q, u[p]); stop if r == n, else p = r

emit(c, v) appends c if v > 127 else -c.
"""
import numpy as np


def u8_column(data) -> np.ndarray:
    """convert_to(np.uint8)[:, 0] of an (n, 2) capture, in the reference's numpy arithmetic (IQArray.py:127-200)"""
    x = np.asarray(data)[:, 0]
    if x.dtype == np.uint8:
        return x.copy()
    if x.dtype == np.int8:
        return np.add(x, 128, dtype=np.uint8, casting="unsafe")
    if x.dtype == np.uint16:
        return (x >> 8).astype(np.uint8)
    if x.dtype == np.int16:
        return (np.add(x, 32768, dtype=np.uint16, casting="unsafe") >> 8).astype(np.uint8)
    with np.errstate(invalid="ignore"):
        return np.multiply(np.add(x, 1.0, dtype=np.float32), 127, dtype=np.float32).astype(np.uint8)


def sub_entries(u) -> list:
    """the reference's `arr` for the uint8 column u (len(u) >= 1)"""
    u = np.asarray(u, dtype=np.uint8)
    n = len(u)
    starts = np.flatnonzero(np.r_[True, u[1:] != u[:-1]])
    run_end = np.repeat(np.r_[starts[1:], n], np.diff(np.r_[starts, n]))   # end of the run holding each position
    order = np.argsort(u, kind="stable")
    nxt = np.full(n, n, np.int64)                                          # next position holding the same value (n: none)
    same = u[order[1:]] == u[order[:-1]]
    nxt[order[:-1][same]] = order[1:][same]
    out = []
    p = 0
    while True:
        v = int(u[p])
        q = int(nxt[p])
        if q == n:
            out.append(1 if v > 127 else -1)
            return out
        r = int(run_end[q])
        c = 1 + r - q
        out.append(c if v > 127 else -c)
        if r == n:
            return out
        p = r


def sub_body(entries) -> bytes:
    """the bytes the reference writes after "Protocol: RAW" and before the final newline"""
    parts = []
    for idx, v in enumerate(entries):
        parts.append(("\nRAW_Data: %d" if idx % 512 == 0 else " %d") % v)
    return "".join(parts).encode()


def sub_header(frequency=433920000, preset="FuriHalSubGhzPresetOok650Async") -> str:
    return "Filetype: Flipper SubGhz RAW File\nVersion: 1\nFrequency: {}\nPreset: {}\nProtocol: RAW".format(frequency, preset)


def sub_file(u, frequency=433920000, preset="FuriHalSubGhzPresetOok650Async") -> bytes:
    return sub_header(frequency, preset).encode() + sub_body(sub_entries(u)) + b"\n"


def body_bound(n: int) -> int:
    """the most body bytes n samples can give (urh_sub_export_bound): every entry but the last covers at least 2 samples"""
    return (3 * n + 3) // 2 + 10 * ((n // 2 + 1 + 511) // 512) + 48
