"""srtb_b200 — thin ctypes binding over libsrtb_b200.so (the C ABI in include/srtb_b200.h).

This is plumbing for tests and bench.py: device memory comes from torch, every data-path
call goes straight into the CUDA library. There is no Python or CPU fallback: if the
library is missing or no CUDA device is present, loading / ctx creation raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE.parent / "csrc" / os.environ.get("SRTB_B200_LIB", "libsrtb_b200.so")  # experiments may build variants

FORMAT_SIMPLE, FORMAT_INTERLEAVED_2, FORMAT_NAOCPSR_SNAP1, FORMAT_GZNUPSR_A1_2, FORMAT_GZNUPSR_A1_4 = range(5)
WINDOW_RECTANGLE, WINDOW_HANN, WINDOW_HAMMING = range(3)
MAX_BOXCARS = 32

# names follow the reference's registry (io/backend_registry.hpp:36-181; unpack_pipe.hpp:392-413)
FORMAT_BY_NAME = {
    "simple": FORMAT_SIMPLE,
    "fastmb_roach2": FORMAT_SIMPLE,
    "interleaved_samples_2": FORMAT_INTERLEAVED_2,
    "naocpsr_snap1": FORMAT_NAOCPSR_SNAP1,
    "gznupsr_a1": FORMAT_GZNUPSR_A1_2,
    "gznupsr_a1_4": FORMAT_GZNUPSR_A1_4,
}
FORMAT_STREAMS = {FORMAT_SIMPLE: 1, FORMAT_INTERLEAVED_2: 2, FORMAT_NAOCPSR_SNAP1: 2,
                  FORMAT_GZNUPSR_A1_2: 2, FORMAT_GZNUPSR_A1_4: 4}


class DetectResult(C.Structure):
    _fields_ = [
        ("zero_count", C.c_uint64),
        ("time_series_count", C.c_uint64),
        ("detect_enabled", C.c_int32),
        ("n_boxcars", C.c_int32),
        ("boxcar_length", C.c_uint64 * MAX_BOXCARS),
        ("series_length", C.c_uint64 * MAX_BOXCARS),
        ("signal_count", C.c_uint64 * MAX_BOXCARS),
        ("variance", C.c_float * MAX_BOXCARS),
        ("threshold", C.c_float * MAX_BOXCARS),
    ]


class BlockConfig(C.Structure):
    _fields_ = [
        ("baseband_input_count", C.c_uint64),
        ("baseband_input_bits", C.c_int32),
        ("baseband_format", C.c_int32),
        ("window", C.c_int32),
        ("baseband_reserve_sample", C.c_int32),
        ("baseband_freq_low", C.c_float),
        ("baseband_bandwidth", C.c_float),
        ("baseband_sample_rate", C.c_float),
        ("dm", C.c_float),
        ("mitigate_rfi_average_method_threshold", C.c_float),
        ("mitigate_rfi_spectral_kurtosis_threshold", C.c_float),
        ("spectrum_channel_count", C.c_uint64),
        ("signal_detect_signal_noise_threshold", C.c_float),
        ("signal_detect_channel_threshold", C.c_float),
        ("signal_detect_max_boxcar_length", C.c_uint64),
        ("rfi_freq_pairs", C.POINTER(C.c_float)),
        ("n_rfi_freq_pairs", C.c_uint64),
    ]


class BlockOutputs(C.Structure):
    """srtb_b200_block_outputs: caller-owned outputs of a ring submission (members may be NULL)"""
    _fields_ = [("d_spectrum", C.c_void_p * 4), ("h_series", C.c_void_p)]


class SrtbError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"srtb_b200 error {code}: {message}")
        self.code = code
        self.message = message


# every symbol include/srtb_b200.h declares: (name, restype, argtypes)
_P, _SZ, _F, _I = C.c_void_p, C.c_size_t, C.c_float, C.c_int
SYMBOLS = {
    "srtb_b200_ctx_create": (_I, [_I, _P, C.POINTER(_P)]),
    "srtb_b200_ctx_destroy": (_I, [_P]),
    "srtb_b200_ctx_set_stream": (_I, [_P, _P]),
    "srtb_b200_synchronize": (_I, [_P]),
    "srtb_b200_last_error": (C.c_char_p, [_P]),
    "srtb_b200_launch_count": (C.c_uint64, [_P]),
    "srtb_b200_version": (C.c_char_p, []),
    "srtb_b200_stage_stats_enable": (C.c_int, [_P, C.c_int]),
    "srtb_b200_stage_stats": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "srtb_b200_unpack": (_I, [_P, _P, _SZ, _I, _I, _I, C.POINTER(_P), _SZ]),
    "srtb_b200_fft_r2c_inplace": (_I, [_P, _P, _SZ]),
    "srtb_b200_fft_c2c": (_I, [_P, _P, _SZ, _SZ, _I]),
    "srtb_b200_watfft_c2c_backward": (_I, [_P, _P, _SZ, _SZ]),
    "srtb_b200_rfi_s1": (_I, [_P, _P, _SZ, _F, _F, C.POINTER(_SZ), _SZ, _P]),
    "srtb_b200_norm_coefficient": (_F, [_SZ, _SZ]),
    "srtb_b200_eval_rfi_ranges": (_SZ, [C.c_char_p, C.POINTER(_F), _SZ]),
    "srtb_b200_rfi_range_to_bins": (_I, [_F, _F, _F, _F, _SZ, C.POINTER(_SZ), C.POINTER(_SZ)]),
    "srtb_b200_dedisperse": (_I, [_P, _P, _SZ, _F, _F, _F, _F]),
    "srtb_b200_nsamps_reserved": (_SZ, [_SZ, _SZ, _F, _F, _F, _F, _I]),
    "srtb_b200_rfi_s2_sk": (_I, [_P, _P, _SZ, _SZ, _F, _P]),
    "srtb_b200_signal_detect": (_I, [_P, _P, _SZ, _SZ, _SZ, _F, _F, _SZ, C.POINTER(DetectResult), _P, _I]),
    "srtb_b200_rfi_sk_v1": (_I, [_P, _P, _SZ, _SZ, _F, _P]),
    "srtb_b200_signal_detect_v1": (_I, [_P, _P, _SZ, _SZ, _F, _F, _F, _SZ, C.POINTER(DetectResult), _P, _I]),
    "srtb_b200_process_block": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, C.POINTER(DetectResult), _P, _I]),
    "srtb_b200_process_block_device": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, C.POINTER(DetectResult), _P, _I]),
    "srtb_b200_process_block_dm_sweep": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, _I, C.POINTER(_F), _SZ,
                                              C.POINTER(DetectResult)]),
    "srtb_b200_submit_block": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ]),
    "srtb_b200_submit_block_device": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ]),
    "srtb_b200_collect_block": (_I, [_P, _I, C.POINTER(DetectResult)]),
    "srtb_b200_submit_block_ex": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, _I, C.POINTER(BlockOutputs)]),
    "srtb_b200_collect_block_ex": (_I, [_P, _I, C.POINTER(DetectResult), C.POINTER(_P), C.POINTER(_P)]),
    "srtb_b200_debug_set_submit_count": (_I, [_P, C.c_uint64]),
    "srtb_b200_block_spectrum": (_P, [_P, _I]),
    "srtb_b200_sweep_spectrum": (_P, [_P]),
}

_lib = None


def load_library(path: os.PathLike | None = None) -> C.CDLL:
    """dlopen libsrtb_b200.so and bind every declared symbol. Raises if it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else LIB_PATH
    if not p.exists():
        raise FileNotFoundError(
            f"{p} not found: build it with __graft_entry__.build() "
            "(simple-radio-telescope-backend_b200/csrc/build.sh). There is no CPU fallback.")
    lib = C.CDLL(str(p))
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def _ptr(t) -> int:
    """device/host pointer of a torch tensor, numpy array or raw int"""
    if t is None:
        return None
    if isinstance(t, int):
        return t
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    if hasattr(t, "ctypes"):
        return t.ctypes.data
    raise TypeError(type(t))


class Context:
    """One srtb_b200_ctx: one GPU, one CUDA stream (replaces the reference's sycl::queue)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.srtb_b200_ctx_create(device, stream, C.byref(h))
        if rc != 0:
            raise SrtbError(rc, self.lib.srtb_b200_last_error(None).decode())
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.srtb_b200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc: int) -> int:
        if rc < 0:
            raise SrtbError(rc, self.lib.srtb_b200_last_error(self.h).decode())
        return rc

    # -- plumbing
    def set_stream(self, stream: int | None):
        self._ck(self.lib.srtb_b200_ctx_set_stream(self.h, stream))

    def synchronize(self):
        self._ck(self.lib.srtb_b200_synchronize(self.h))

    @property
    def launch_count(self) -> int:
        return int(self.lib.srtb_b200_launch_count(self.h))

    # -- stages (names follow the reference's pipes)
    def unpack(self, d_in, in_bytes: int, bits: int, fmt: int, window: int, outs, out_count: int):
        arr = (C.c_void_p * 4)(*([_ptr(o) for o in outs] + [None] * (4 - len(outs))))
        self._ck(self.lib.srtb_b200_unpack(self.h, _ptr(d_in), in_bytes, bits, fmt, window, arr, out_count))

    def fft_r2c_inplace(self, d_inout, n_real: int):
        self._ck(self.lib.srtb_b200_fft_r2c_inplace(self.h, _ptr(d_inout), n_real))

    def fft_c2c(self, d_x, length: int, batch: int, direction: int):
        self._ck(self.lib.srtb_b200_fft_c2c(self.h, _ptr(d_x), length, batch, direction))

    def watfft_c2c_backward(self, d_x, length: int, batch: int):
        self._ck(self.lib.srtb_b200_watfft_c2c_backward(self.h, _ptr(d_x), length, batch))

    def rfi_s1(self, d_x, count: int, avg_threshold: float, norm_coef: float, bin_ranges=(), d_mean_out=None):
        n = len(bin_ranges)
        flat = (C.c_size_t * (2 * n))(*[v for r in bin_ranges for v in r]) if n else None
        self._ck(self.lib.srtb_b200_rfi_s1(self.h, _ptr(d_x), count, avg_threshold, norm_coef, flat, n,
                                           _ptr(d_mean_out)))

    def dedisperse(self, d_x, count: int, f_min: float, f_c: float, df: float, dm: float):
        self._ck(self.lib.srtb_b200_dedisperse(self.h, _ptr(d_x), count, f_min, f_c, df, dm))

    def rfi_s2_sk(self, d_x, time_count: int, chan_count: int, sk_threshold: float, d_sk_out=None):
        self._ck(self.lib.srtb_b200_rfi_s2_sk(self.h, _ptr(d_x), time_count, chan_count, sk_threshold,
                                              _ptr(d_sk_out)))

    def signal_detect(self, d_x, time_count: int, chan_count: int, time_reserved_count: int, snr: float,
                      channel_threshold: float, max_boxcar: int, h_series=None, copy_all: bool = False):
        res = DetectResult()
        self._ck(self.lib.srtb_b200_signal_detect(self.h, _ptr(d_x), time_count, chan_count,
                                                  time_reserved_count, snr, channel_threshold, max_boxcar,
                                                  C.byref(res), _ptr(h_series), int(copy_all)))
        return res

    def rfi_sk_v1(self, d_x, fft_bins: int, time_counts: int, sk_threshold: float, d_sk_out=None):
        """SK v1 on spectra laid out [time][frequency] (reference: spectrum/rfi_mitigation.hpp:181-275)"""
        self._ck(self.lib.srtb_b200_rfi_sk_v1(self.h, _ptr(d_x), fft_bins, time_counts, sk_threshold, _ptr(d_sk_out)))

    def signal_detect_v1(self, d_x, count_per_batch: int, batch_size: int, sk_threshold: float, snr: float,
                         channel_threshold: float, max_boxcar: int, h_series=None, copy_all: bool = False):
        """signal_detect_pipe v1 (reference: pipeline/signal_detect_pipe.hpp:51-230)"""
        res = DetectResult()
        self._ck(self.lib.srtb_b200_signal_detect_v1(self.h, _ptr(d_x), count_per_batch, batch_size, sk_threshold, snr,
                                                     channel_threshold, max_boxcar, C.byref(res), _ptr(h_series),
                                                     int(copy_all)))
        return res

    def stage_stats_enable(self, on: bool = True):
        self._ck(self.lib.srtb_b200_stage_stats_enable(self.h, int(on)))

    def stage_stats(self, stage: int):
        """(ms, algorithmic bytes) of the last call of `stage` (0 unpack .. 6 signal_detect)"""
        ms, nbytes = C.c_double(), C.c_double()
        self._ck(self.lib.srtb_b200_stage_stats(self.h, int(stage), C.byref(ms), C.byref(nbytes)))
        return ms.value, nbytes.value

    def process_block(self, cfg: BlockConfig, baseband, nbytes: int, h_series=None, copy_all: bool = False,
                      on_device: bool = False):
        res = (DetectResult * 4)()
        fn = self.lib.srtb_b200_process_block_device if on_device else self.lib.srtb_b200_process_block
        n = self._ck(fn(self.h, C.byref(cfg), _ptr(baseband), nbytes, res, _ptr(h_series), int(copy_all)))
        return [res[i] for i in range(n)]

    def process_block_dm_sweep(self, cfg: BlockConfig, baseband, nbytes: int, dms, on_device: bool = False):
        """one block, many trial DMs: returns results[dm_index][stream]"""
        n_dm = len(dms)
        arr = (C.c_float * n_dm)(*[float(d) for d in dms])
        res = (DetectResult * (4 * n_dm))()
        streams = self._ck(self.lib.srtb_b200_process_block_dm_sweep(self.h, C.byref(cfg), _ptr(baseband), nbytes,
                                                                      int(on_device), arr, n_dm, res))
        return [[res[j * streams + s] for s in range(streams)] for j in range(n_dm)]

    def submit_block(self, cfg: BlockConfig, h_baseband, nbytes: int) -> int:
        """pipelined ingest: H2D on the copy stream overlaps the previous block's compute"""
        return self._ck(self.lib.srtb_b200_submit_block(self.h, C.byref(cfg), _ptr(h_baseband), nbytes))

    def submit_block_device(self, cfg: BlockConfig, d_baseband, nbytes: int) -> int:
        return self._ck(self.lib.srtb_b200_submit_block_device(self.h, C.byref(cfg), _ptr(d_baseband), nbytes))

    def collect_block(self, ticket: int):
        res = (DetectResult * 4)()
        n = self._ck(self.lib.srtb_b200_collect_block(self.h, ticket, res))
        return [res[i] for i in range(n)]

    def submit_block_ex(self, cfg: BlockConfig, baseband, nbytes: int, on_device: bool = False, d_spectrum=None,
                        h_series=None) -> int:
        """ring submission with caller-owned outputs: d_spectrum = per-stream device buffers of N + 2 floats (the
        dynamic spectrum stays there), h_series = pinned host buffer [streams][MAX_BOXCARS][L] for positive series"""
        out = BlockOutputs()
        for i, t in enumerate(d_spectrum or []):
            out.d_spectrum[i] = _ptr(t)
        out.h_series = _ptr(h_series)
        return self._ck(self.lib.srtb_b200_submit_block_ex(self.h, C.byref(cfg), _ptr(baseband), nbytes,
                                                           int(on_device), C.byref(out)))

    def collect_block_ex(self, ticket: int):
        """(results, host pointer of the series buffer, [device pointers of the streams' dynamic spectra])"""
        res = (DetectResult * 4)()
        series = C.c_void_p()
        spec = (C.c_void_p * 4)()
        n = self._ck(self.lib.srtb_b200_collect_block_ex(self.h, ticket, res, C.byref(series), spec))
        return [res[i] for i in range(n)], series.value, [spec[i] for i in range(n)]

    def debug_set_submit_count(self, value: int):
        self._ck(self.lib.srtb_b200_debug_set_submit_count(self.h, value))

    def block_spectrum_ptr(self, stream: int) -> int:
        return self.lib.srtb_b200_block_spectrum(self.h, stream)

    def sweep_spectrum_ptr(self) -> int:
        """test hook: device pointer of the last trial's dynamic spectrum (last stream) of the latest DM sweep"""
        return self.lib.srtb_b200_sweep_spectrum(self.h)


# host helpers (pure host arithmetic of the reference's pipes)
def norm_coefficient(in_count: int, channel_count: int) -> float:
    return float(load_library().srtb_b200_norm_coefficient(in_count, channel_count))


def eval_rfi_ranges(freq_list: str):
    lib = load_library()
    buf = (C.c_float * 128)()
    n = lib.srtb_b200_eval_rfi_ranges(freq_list.encode(), buf, 64)
    return [(buf[2 * i], buf[2 * i + 1]) for i in range(min(n, 64))]


def rfi_range_to_bins(f1: float, f2: float, freq_low: float, bandwidth: float, in_count: int):
    lib = load_library()
    lo, hi = C.c_size_t(), C.c_size_t()
    ok = lib.srtb_b200_rfi_range_to_bins(f1, f2, freq_low, bandwidth, in_count, C.byref(lo), C.byref(hi))
    return (lo.value, hi.value) if ok else None


def nsamps_reserved(baseband_input_count: int, channel_count: int, freq_low: float, bandwidth: float,
                    sample_rate: float, dm: float, reserve_sample: bool) -> int:
    return int(load_library().srtb_b200_nsamps_reserved(baseband_input_count, channel_count, freq_low,
                                                         bandwidth, sample_rate, dm, int(reserve_sample)))
