"""ctypes binding of liburh_b200.so (the C ABI declared in include/urh_b200.h).

There is NO CPU fallback: if the shared library is missing or no CUDA device is present, every
entry point raises (``UrhCudaUnavailable``).  Importing this module never touches the GPU; the
context is created lazily on first use.
"""
import ctypes as C
import os
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("URH_B200_LIB", os.path.join(HERE, "liburh_b200.so"))

URH_OK = 0
ERR_CUDA, ERR_INVALID, ERR_DTYPE, ERR_NOMEM, ERR_MODULATION, ERR_NO_DEVICE = -1, -2, -3, -4, -5, -6

DT_I8, DT_U8, DT_I16, DT_U16, DT_F32 = 0, 1, 2, 3, 4
MOD_ASK, MOD_FSK, MOD_PSK, MOD_QAM, MOD_GFSK, MOD_OQPSK = 0, 1, 2, 3, 4, 5
# streamed entry points (include/urh_b200.h)
STREAM_AFP_DEMOD, STREAM_GRAB_PULSE_LENS, STREAM_DEMOD_DIGITIZE, STREAM_DEMOD_CENTER_DIGITIZE = 0, 1, 2, 3
STREAM_QAD_OUT, STREAM_RESIDENT, STREAM_QAD_ON_DEVICE = 0x10, 0x20, 0x40
STREAM_PSK, STREAM_PSK4 = 0x80, 0x100
STREAM_UPLOAD, STREAM_DOWNLOAD, STREAM_HALO = 1, 2, 4

_DTYPE_CODE = {
    np.dtype(np.int8): DT_I8,
    np.dtype(np.uint8): DT_U8,
    np.dtype(np.int16): DT_I16,
    np.dtype(np.uint16): DT_U16,
    np.dtype(np.float32): DT_F32,
}
_CODE_DTYPE = {v: k for k, v in _DTYPE_CODE.items()}


class UrhCudaUnavailable(RuntimeError):
    """The CUDA library or a CUDA device is missing; the product path has no CPU fallback."""


def dtype_code(dtype) -> int:
    try:
        return _DTYPE_CODE[np.dtype(dtype)]
    except (KeyError, TypeError):
        raise ValueError("Unsupported dtype")


def demod_mod_code(mod_type: str) -> int:
    """mod_type string of afp_demod / grab_pulse_lens -> code (anything unknown behaves like the
    reference: afp_demod leaves zeros, NOISE sentinel 0)."""
    return {"ASK": MOD_ASK, "FSK": MOD_FSK, "PSK": MOD_PSK, "QAM": MOD_QAM, "OQPSK": MOD_OQPSK}.get(mod_type, -1)


_lib = None
_lib_lock = threading.Lock()

i64, i32, u16, u32, u8, f32, vp = C.c_int64, C.c_int, C.c_uint16, C.c_uint32, C.c_uint8, C.c_float, C.c_void_p
szt = C.c_size_t

# name -> (restype, argtypes); every symbol declared in include/urh_b200.h must be listed here
# (tests/test_abi.py checks header <-> library <-> this table).
SIGNATURES = {
    "urh_device_count": (i32, []),
    "urh_ctx_create": (i32, [i32, C.POINTER(vp)]),
    "urh_ctx_destroy": (None, [vp]),
    "urh_last_error": (C.c_char_p, [vp]),
    "urh_sync": (i32, [vp]),
    "urh_device_info": (i32, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(szt), C.c_char_p, i32]),
    "urh_malloc": (i32, [vp, szt, C.POINTER(vp)]),
    "urh_free": (i32, [vp, vp]),
    "urh_memset": (i32, [vp, vp, i32, szt]),
    "urh_memcpy_h2d": (i32, [vp, vp, vp, szt]),
    "urh_memcpy_d2h": (i32, [vp, vp, vp, szt]),
    "urh_memcpy_d2d": (i32, [vp, vp, vp, szt]),
    "urh_host_alloc": (i32, [vp, szt, C.POINTER(vp)]),
    "urh_host_free": (i32, [vp, vp]),
    "urh_timer_start": (i32, [vp]),
    "urh_timer_stop": (i32, [vp, C.POINTER(f32)]),
    "urh_timeline_fetch": (i32, [vp, vp, vp, i32, C.POINTER(i32)]),
    "urh_launch_count": (i64, [vp]),
    "urh_afp_demod": (i32, [vp, vp, i32, i64, f32, i32, i32, f32, vp]),
    "urh_get_center_thresholds": (i32, [f32, f32, i32, vp]),
    "urh_grab_pulse_lens": (i32, [vp, vp, i64, f32, u16, i32, u32, u8, f32, C.POINTER(i64)]),
    "urh_demod_digitize": (i32, [vp, vp, i32, i64, f32, i32, f32, u16, u32, u8, f32, vp, C.POINTER(i64)]),
    "urh_fetch_pulses": (i32, [vp, vp, i64]),
    "urh_pulses_device_ptr": (i32, [vp, C.POINTER(vp), C.POINTER(i64)]),
    "urh_get_magnitudes": (i32, [vp, vp, i32, i64, vp]),
    "urh_noise_chunk_stats_iq": (i32, [vp, vp, i32, i64, i64, i32, vp, vp]),
    "urh_noise_chunk_stats": (i32, [vp, vp, i32, i64, i64, i32, vp, vp]),
    "urh_center_stats": (i32, [vp, vp, i64, i64, vp]),
    "urh_center_histogram": (i32, [vp, vp, i64, i64, i64, C.c_double, C.c_double, i64, vp]),
    "urh_afp_demod_tiles": (i32, [vp, vp, i32, i64, f32, i32, vp, i32, vp]),
    "urh_center_window_stats": (i32, [vp, vp, i64, i64, i64, vp]),
    "urh_center_window_var": (i32, [vp, vp, i64, i64, i64, vp]),
    "urh_center_histogram_tiles": (i32, [vp, vp, i64, i64, i64, C.c_double, C.c_double, i64, vp]),
    "urh_segment_messages": (i32, [vp, vp, i32, i64, f32, vp, i64, C.POINTER(i64)]),
    "urh_plateau_lengths": (i32, [vp, vp, i64, f32, i32, vp, i64, C.POINTER(i64)]),
    "urh_median_filter": (i32, [vp, vp, i64, C.c_uint, vp]),
    "urh_arr2decibel": (i32, [vp, vp, i64, vp]),
    "urh_modulate_batch": (i32, [vp, vp, vp, vp, i32, u32, i32, vp, i32, i32, f32, f32, f32, f32, u32, i32, vp, i32, vp]),
    "urh_fir_filter": (i32, [vp, vp, i64, vp, i32, vp]),
    "urh_convolve_c128": (i32, [vp, vp, i64, vp, i32, i64, i64, vp]),
    "urh_dc_correction": (i32, [vp, vp, i64, vp, i32]),
    "urh_dc_correction_int": (i32, [vp, vp, i32, i64, vp]),
    "urh_fir_filter_shard": (i32, [vp, vp, i64, i32, vp, i32, vp]),
    "urh_dc_column_sums": (i32, [vp, vp, i64, i32, vp, vp]),
    "urh_dc_subtract": (i32, [vp, vp, i64, f32, f32, vp]),
    "urh_dc_int_column_sums": (i32, [vp, vp, i32, i64, vp]),
    "urh_dc_int_subtract": (i32, [vp, vp, i32, i64, C.c_double, C.c_double, vp]),
    "urh_stft": (i32, [vp, vp, i64, i32, i32, vp, i64, vp]),
    "urh_spectrogram_db": (i32, [vp, vp, i64, i32, i32, vp, i64, vp]),
    "urh_shard_dense": (i32, [vp, vp, i32, i64, i32, f32, i32, f32, u16, u8, f32, vp, vp]),
    "urh_shard_dense_qad": (i32, [vp, vp, i64, i32, f32, u16, u8, f32, vp]),
    "urh_shard_candidates": (i32, [vp, i32, i32, i64, i64, C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(i32)]),
    "urh_shard_fire": (i32, [vp, i32, C.POINTER(i64), C.POINTER(i64)]),
    "urh_shard_rows": (i32, [vp, i64, u16, i32, u32, i64, i32, C.POINTER(i64)]),
    "urh_nccl_allgather_host": (i32, [vp, vp, vp, szt]),
    "urh_nccl_allreduce_host_i64": (i32, [vp, vp, i64, i32]),
    "urh_p2p_create": (i32, [vp, vp]),
    "urh_p2p_open": (i32, [vp, vp, i32, i32]),
    "urh_p2p_close": (i32, [vp]),
    "urh_p2p_allgather_host": (i32, [vp, vp, vp, szt]),
    "urh_p2p_allgather_dev": (i32, [vp, vp, vp, szt]),
    "urh_p2p_allreduce_u64_dev": (i32, [vp, vp, vp, vp, i32]),
    "urh_p2p_check": (i32, [vp]),
    "urh_demod_center_digitize": (i32, [vp, vp, i32, i64, f32, i32, u16, u32, i64, vp, C.POINTER(C.c_double), C.POINTER(i32), C.POINTER(i64)]),
    "urh_demod_center_digitize_host": (i32, [vp, vp, i32, i64, f32, i32, u16, u32, i64, i64, vp, vp, C.POINTER(C.c_double), C.POINTER(i32),
                                             C.POINTER(i64)]),
    "urh_shard_demod_center_digitize_host": (i32, [vp, vp, i32, i64, i32, f32, i32, u16, u32, i64, i64, vp, vp, i64, i64, C.POINTER(C.c_double),
                                                   C.POINTER(i32), C.POINTER(i64)]),
    "urh_shard_demod_center_digitize": (i32, [vp, vp, i32, i64, i32, f32, i32, u16, u32, i64, vp, i64, i64, C.POINTER(C.c_double),
                                              C.POINTER(i32), C.POINTER(i64)]),
    "urh_shard_digitize": (i32, [vp, vp, i32, vp, i64, i32, f32, i32, f32, u16, u32, u8, f32, vp, i64, i64, C.POINTER(i64)]),
    "urh_segment_shard_pass": (i32, [vp, vp, i32, i64, f32, vp]),
    "urh_segments_from_runs": (i32, [vp, vp, i64, i32, i32, i64, i64, vp, i64, C.POINTER(i64)]),
    "urh_fetch_candidates": (i32, [vp, vp, vp, i64]),
    "urh_pulses_from_table": (i32, [vp, vp, vp, i64, i64, u16, i32, u32, i32, C.POINTER(i64)]),
    "urh_costas_halo_samples": (i32, []),
    "urh_costas_shard_speculate": (i32, [vp, vp, i32, i64, i32, f32, i32, f32, vp]),
    "urh_costas_shard_resolve": (i32, [vp, vp, vp]),
    "urh_fft_argmax": (i32, [vp, vp, i64, vp, vp]),
    "urh_convert_iq": (i32, [vp, vp, i32, vp, i32, i64]),
    "urh_modulation_features": (i32, [vp, vp, i64, i32, i32, vp, vp]),
    "urh_cwt_haar": (i32, [vp, vp, i32, i64, i32, vp, vp]),
    "urh_ppseq_to_bits": (i32, [vp, vp, i64, u32, u8, i32, i32, vp, vp, vp]),
    "urh_fetch_bits": (i32, [vp, vp, vp, vp, vp]),
    "urh_bits_device_ptr": (vp, [vp]),
    "urh_nccl_unique_id": (i32, [vp]),
    "urh_nccl_init": (i32, [vp, vp, i32, i32]),
    "urh_nccl_destroy": (i32, [vp]),
    "urh_nccl_allreduce_f64": (i32, [vp, vp, i64, i32]),
    "urh_nccl_allreduce_i64": (i32, [vp, vp, i64, i32]),
    "urh_nccl_allgather": (i32, [vp, vp, vp, szt]),
    "urh_nccl_gatherv": (i32, [vp, vp, vp, vp, i32]),
    "urh_nccl_sendrecv": (i32, [vp, vp, szt, i32, vp, szt, i32]),
    "urh_set_profiling": (i32, [vp, i32]),
    "urh_last_dense_ms": (i32, [vp, C.POINTER(f32)]),
    "urh_costas_shard_hypotheses": (i32, [vp, vp, C.POINTER(i32)]),
    "urh_costas_shard_adopt": (i32, [vp, i32, vp]),
    "urh_costas_stats": (i32, [vp, vp]),
    "urh_center_certify_stats": (i32, [vp, vp]),
    "urh_speculate_stats": (i32, [vp, vp]),
    "urh_costas_last_redone": (i64, [vp]),
    "urh_costas_stitch_stats": (i32, [vp, vp]),
    "urh_selftest_packed_div": (i32, [vp, C.c_uint64, i64, C.POINTER(i64), C.POINTER(i64)]),
    "urh_bgra_lookup": (i32, [vp, vp, i64, i64, vp, i32, f32, f32, i32, vp]),
    "urh_spectrogram_bgra": (i32, [vp, vp, i64, i32, i32, vp, vp, vp, i32, vp, i32, f32, f32, i32, vp]),
    "urh_gather_samples": (i32, [vp, vp, i64, i64, i64, i64, vp]),
    "urh_fta_records": (i32, [vp, vp, i64, i32, i64, i64, vp, C.c_double, i32, vp, vp]),
    "urh_path_minmax": (i32, [vp, vp, i32, i64, i64, i64, i64, i64, vp]),
    "urh_qpath_streams": (i32, [vp, vp, i32, i64, i64, i64, i64, i64, i64, vp, vp, i32, vp, vp]),
    "urh_modulate_stats": (i32, [vp, vp]),
    "urh_synth_psk": (i32, [vp, vp, i64, i64, i32, i32, C.c_double, f32, f32, C.c_uint64, i64, i64, i64]),
    "urh_afp_demod_stream": (i32, [vp, vp, i32, i64, f32, i32, i64, i32, vp]),
    "urh_grab_pulse_lens_stream": (i32, [vp, vp, i32, i64, f32, u16, i32, u32, u8, f32, i64, i32, C.POINTER(i64)]),
    "urh_demod_digitize_stream": (i32, [vp, vp, i32, i64, f32, i32, f32, u16, u32, u8, f32, i64, i32, vp, C.POINTER(i64)]),
    "urh_demod_center_digitize_stream": (i32, [vp, vp, i32, i64, f32, i32, u16, u32, i64, i64, i32, vp, vp, C.POINTER(C.c_double),
                                               C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]),
    "urh_afp_demod_psk_stream": (i32, [vp, vp, i32, i64, f32, i32, f32, i64, i32, vp]),
    "urh_demod_digitize_psk_stream": (i32, [vp, vp, i32, i64, f32, f32, u16, u32, u8, f32, i64, i32, vp, C.POINTER(i64)]),
    "urh_stream_footprint": (i32, [i64, i32, i32, i64, i32, i32, i64, C.POINTER(i64)]),
    "urh_stream_schedule": (i32, [i64, i64, i32, i32, vp, i64, C.POINTER(i64)]),
    "urh_stream_stats": (i32, [vp, vp]),
    "urh_mem_get_info": (i32, [vp, C.POINTER(szt), C.POINTER(szt)]),
    "urh_synth_fsk": (i32, [vp, vp, i64, i64, i32, vp, vp, C.c_double, f32, f32, C.c_uint64, i64, i64, i64, i64, i64]),
}


def load_library():
    """dlopen liburh_b200.so and declare all prototypes (no GPU needed)."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise UrhCudaUnavailable(
                "liburh_b200.so not built (run `python -m urh_b200.build`); there is no CPU fallback"
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


class Context:
    """One CUDA device + stream + scratch arena (urh_ctx)."""

    def __init__(self, device: int = 0):
        self.lib = load_library()
        h = vp()
        rc = self.lib.urh_ctx_create(int(device), C.byref(h))
        if rc == ERR_NO_DEVICE:
            raise UrhCudaUnavailable("no CUDA device visible; urh_b200 has no CPU fallback")
        if rc != URH_OK:
            raise RuntimeError("urh_ctx_create(device=%d) failed: %d" % (device, rc))
        self.handle = h
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.urh_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- error mapping (same exception types the reference raises) --
    def check(self, rc: int):
        if rc == URH_OK:
            return
        msg = self.lib.urh_last_error(self.handle)
        msg = msg.decode(errors="replace") if msg else ""
        if rc == ERR_DTYPE:
            raise ValueError(msg or "Unsupported dtype")
        if rc == ERR_INVALID:
            raise ValueError(msg)
        if rc == ERR_MODULATION:
            raise AssertionError(msg)
        if rc == ERR_NOMEM:
            raise MemoryError(msg)
        raise RuntimeError("urh_b200 error %d: %s" % (rc, msg))

    def sync(self):
        self.check(self.lib.urh_sync(self.handle))

    def launch_count(self) -> int:
        return int(self.lib.urh_launch_count(self.handle))

    def device_info(self) -> dict:
        sm, ma, mi, tot = i32(), i32(), i32(), szt()
        name = C.create_string_buffer(256)
        self.check(self.lib.urh_device_info(self.handle, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(tot), name, 256))
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "total_mem": tot.value, "name": name.value.decode()}

    def timer_start(self):
        self.check(self.lib.urh_timer_start(self.handle))

    def timer_stop(self) -> float:
        ms = f32()
        self.check(self.lib.urh_timer_stop(self.handle, C.byref(ms)))
        return float(ms.value)


_default_ctx = {}
_ctx_lock = threading.Lock()


def default_context(device: int = None) -> Context:
    """Process-wide context per device (device defaults to $URH_B200_DEVICE, $LOCAL_RANK or 0)."""
    if device is None:
        device = int(os.environ.get("URH_B200_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    with _ctx_lock:
        ctx = _default_ctx.get(device)
        if ctx is None:
            ctx = Context(device)
            _default_ctx[device] = ctx
        return ctx


def cuda_available() -> bool:
    try:
        return load_library().urh_device_count() > 0
    except (UrhCudaUnavailable, OSError):
        return False
