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
RING_SLOTS = 3  # SRTB_B200_RING_SLOTS: blocks the ring keeps in flight

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
        # non-zero: one more result per block, the detector on the streams' total intensity (include/srtb_b200.h)
        ("signal_detect_sum_streams", C.c_int32),
    ]


class BlockOutputs(C.Structure):
    """srtb_b200_block_outputs: caller-owned outputs of a ring submission (members may be NULL)"""
    _fields_ = [("d_spectrum", C.c_void_p * 4), ("h_series", C.c_void_p)]


class Peak(C.Structure):
    """srtb_b200_peak: per boxcar, the series' peak S/N and the first index of its maximum"""
    _fields_ = [("snr", C.c_float * MAX_BOXCARS), ("peak_index", C.c_uint64 * MAX_BOXCARS)]


class SweepOutputs(C.Structure):
    """srtb_b200_sweep_outputs: what a DM sweep hands out besides its result headers (members may be NULL)"""
    _fields_ = [("h_peaks", C.c_void_p), ("h_best_trial", C.c_void_p), ("h_series", C.c_void_p),
                ("d_spectrum", C.c_void_p * 4)]


class Event(C.Structure):
    """srtb_b200_event: one above-threshold run [begin, end) of one boxcar series of one trial and stream"""
    _fields_ = [("begin", C.c_uint64), ("end", C.c_uint64), ("peak_index", C.c_uint64), ("snr", C.c_float),
                ("trial", C.c_uint32), ("boxcar", C.c_uint32), ("stream", C.c_uint32)]


class Candidate(C.Structure):
    """srtb_b200_candidate: one friends-of-friends group of events (srtb_b200_cluster_events)"""
    _fields_ = [("snr", C.c_float), ("dm", C.c_float), ("dm_low", C.c_float), ("dm_high", C.c_float),
                ("boxcar_length", C.c_uint64), ("peak_index", C.c_uint64), ("window", C.c_uint64),
                ("members", C.c_uint64), ("span_begin", C.c_uint64), ("span_end", C.c_uint64),
                ("trial", C.c_uint32), ("stream", C.c_uint32)]


class CutoutRequest(C.Structure):
    """srtb_b200_cutout_request: one candidate's cut-out (srtb_b200_candidate_cutouts): the spectrum sample at the
    image's bin W/2, the image's DM, the plane's DM half-width and the decimation q"""
    _fields_ = [("center", C.c_int64), ("dm", C.c_float), ("dm_halfwidth", C.c_float), ("decimation", C.c_uint32)]


def _dtype_of(struct):
    """the numpy structured dtype with struct's field names, offsets and size"""
    import numpy as np
    names, formats, offsets = [], [], []
    for name, ctype in struct._fields_:
        names.append(name)
        formats.append(np.dtype(ctype))
        offsets.append(getattr(struct, name).offset)
    return np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": C.sizeof(struct)})


class SrtbError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"srtb_b200 error {code}: {message}")
        self.code = code
        self.message = message


# waterfall thumbnail colours (srtb::gui, include/srtb/config.hpp)
GUI_OPAQUE = 0xFF000000
GUI_COLOR_0 = 0xFF1F1E33
GUI_COLOR_1 = 0xFF33E1F1
GUI_COLOR_OVERFLOW = 0xFFE0E1CC

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
    "srtb_b200_process_block_dm_sweep_ex": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, _I, C.POINTER(_F), _SZ,
                                                 C.POINTER(DetectResult), C.POINTER(SweepOutputs)]),
    "srtb_b200_submit_block": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ]),
    "srtb_b200_submit_block_device": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ]),
    "srtb_b200_collect_block": (_I, [_P, _I, C.POINTER(DetectResult)]),
    "srtb_b200_submit_block_ex": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, _I, C.POINTER(BlockOutputs)]),
    "srtb_b200_collect_block_ex": (_I, [_P, _I, C.POINTER(DetectResult), C.POINTER(_P), C.POINTER(_P)]),
    "srtb_b200_debug_set_submit_count": (_I, [_P, C.c_uint64]),
    "srtb_b200_block_spectrum": (_P, [_P, _I]),
    "srtb_b200_sweep_spectrum": (_P, [_P]),
    "srtb_b200_simplify_spectrum": (_I, [_P, _P, _SZ, _SZ, _SZ, _SZ, C.c_uint32, C.c_uint32, C.c_uint32, _P, _P, _P]),
    "srtb_b200_cross_spectrum": (_I, [_P, _P, _P, _SZ, _F, _P]),
    "srtb_b200_correlate": (_I, [_P, _P, _P, _SZ, _P]),
    "srtb_b200_correlate_accumulate": (_I, [_P, _P, _P, _I, _SZ, _SZ, _P, _I]),
    "srtb_b200_correlate_finish": (_I, [_P, _P, _SZ, C.c_uint64, _P]),
    "srtb_b200_incoherent_shifts": (_I, [_SZ, _F, _F, _F, _F, C.POINTER(_F), _SZ, _P, C.POINTER(C.c_uint64),
                                         C.POINTER(C.c_uint64)]),
    "srtb_b200_incoherent_groups": (_I, [_SZ, _F, _F, _F, _F, C.POINTER(_F), _SZ, _P, _P, _P, C.POINTER(C.c_uint64),
                                         C.POINTER(C.c_uint32)]),
    "srtb_b200_incoherent_dm_search": (_I, [_P, _P, _SZ, _SZ, _SZ, _F, _F, _F, _F, C.POINTER(_F), _SZ, _F, _F, _SZ,
                                            C.POINTER(DetectResult), _P, _P, _P]),
    "srtb_b200_series_events": (_I, [_P, _P, _SZ, _SZ, C.POINTER(DetectResult), _SZ, _P, _SZ,
                                     C.POINTER(C.c_uint64)]),
    "srtb_b200_incoherent_dm_search_events": (_I, [_P, _P, _SZ, _SZ, _SZ, C.c_float, C.c_float, C.c_float,
                                                   C.c_float, C.POINTER(C.c_float), _SZ, C.c_float, C.c_float, _SZ,
                                                   C.POINTER(DetectResult), _P, _P, _P, _P, _SZ,
                                                   C.POINTER(C.c_uint64)]),
    "srtb_b200_process_block_dm_sweep_events": (_I, [_P, _P, _P, _SZ, _I, C.POINTER(C.c_float), _SZ,
                                                     C.POINTER(DetectResult), _P, _P, _SZ, C.POINTER(C.c_uint64)]),
    "srtb_b200_cluster_events": (_I, [_P, _SZ, C.POINTER(C.c_float), _SZ, _P, _SZ, C.POINTER(C.c_uint64)]),
    "srtb_b200_submit_block_events": (_I, [_P, C.POINTER(BlockConfig), _P, _SZ, _I, C.POINTER(BlockOutputs), _SZ]),
    "srtb_b200_collect_block_events": (_I, [_P, _I, C.POINTER(DetectResult), C.POINTER(_P), C.POINTER(_P),
                                            C.POINTER(_P), C.POINTER(C.c_uint64)]),
    "srtb_b200_candidate_cutouts": (_I, [_P, _P, _I, _SZ, _SZ, _SZ, _F, _F, _F, _F, C.POINTER(CutoutRequest), _SZ,
                                         _SZ, _SZ, _SZ, _P, _P, _P]),
    "srtb_b200_fold_phase": (_I, [C.c_double, C.c_double, C.c_double, C.c_uint64, C.c_uint64,
                                  C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "srtb_b200_fold": (_I, [_P, C.POINTER(_P), _I, _SZ, _SZ, _SZ, C.c_double, C.c_double, C.c_double, _SZ, _SZ,
                            _P, _P, _P]),
    "srtb_b200_fold_coherence": (_I, [_P, _P, _P, _SZ, _SZ, _SZ, C.c_double, C.c_double, C.c_double, _SZ, _SZ,
                                      _P, _P, _P]),
}
INCOHERENT_MAX_DMS = 4096
FOLD_MAX_BINS = 4096

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
        self._sum_tickets = {}  # ring ticket -> submitted with signal_detect_sum_streams
        self._event_caps = {}  # ring ticket -> max_events of submit_block_events

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
        """results per stream, then the total-intensity sum's when cfg.signal_detect_sum_streams is set (h_series then
        has streams + 1 slots)"""
        res = (DetectResult * 5)()
        fn = self.lib.srtb_b200_process_block_device if on_device else self.lib.srtb_b200_process_block
        n = self._ck(fn(self.h, C.byref(cfg), _ptr(baseband), nbytes, res, _ptr(h_series), int(copy_all)))
        return [res[i] for i in range(n + (1 if cfg.signal_detect_sum_streams else 0))]

    def process_block_dm_sweep_events(self, cfg: BlockConfig, baseband, nbytes: int, dms, max_events: int,
                                      on_device: bool = False, h_series=None, d_spectrum=None):
        """process_block_dm_sweep(outputs=True) that also lists every trial's events (srtb_b200_event): returns
        (results, peaks, best_trial, h_series, d_spectrum, events, n_events), events[s] a numpy structured array of
        stream s's first min(n_events[s], max_events) events"""
        return self.process_block_dm_sweep(cfg, baseband, nbytes, dms, on_device, True, h_series, d_spectrum,
                                           max_events=max_events)

    def process_block_dm_sweep(self, cfg: BlockConfig, baseband, nbytes: int, dms, on_device: bool = False,
                               outputs: bool = False, h_series=None, d_spectrum=None, max_events=None):
        """one block, many trial DMs: returns results[dm_index][stream].
        outputs=True: returns (results, peaks, best_trial, h_series, d_spectrum) instead, where peaks = (snr, index),
        numpy arrays [n_dm][streams][n_boxcars] (n_boxcars = the most any trial used), best_trial = [streams] ints,
        h_series = pinned [streams][MAX_BOXCARS][L] float32 tensor holding the best trials' positive series and
        d_spectrum = per-stream device tensors of N + 2 float32 holding the best trials' dynamic spectra. The caller may
        pass h_series and d_spectrum in (the same shapes); they are allocated otherwise."""
        n_dm = len(dms)
        arr = (C.c_float * n_dm)(*[float(d) for d in dms])
        res = (DetectResult * (4 * n_dm))()
        if not outputs:
            streams = self._ck(self.lib.srtb_b200_process_block_dm_sweep(self.h, C.byref(cfg), _ptr(baseband), nbytes,
                                                                          int(on_device), arr, n_dm, res))
            return [[res[j * streams + s] for s in range(streams)] for j in range(n_dm)]
        import numpy as np
        import torch
        streams = FORMAT_STREAMS[cfg.baseband_format]
        n = cfg.baseband_input_count
        L = n // 2 // min(cfg.spectrum_channel_count, n // 2)
        if h_series is None:
            h_series = torch.zeros((streams, MAX_BOXCARS, L), dtype=torch.float32).pin_memory()
        if d_spectrum is None:
            d_spectrum = [torch.empty(n + 2, dtype=torch.float32, device=f"cuda:{self.device}") for _ in range(streams)]
        peaks = (Peak * (4 * n_dm))()
        best = (C.c_int32 * 4)()
        out = SweepOutputs()
        out.h_peaks = C.cast(peaks, C.c_void_p)
        out.h_best_trial = C.cast(best, C.c_void_p)
        out.h_series = _ptr(h_series)
        for i, t in enumerate(d_spectrum):
            out.d_spectrum[i] = _ptr(t)
        if max_events is None:
            streams = self._ck(self.lib.srtb_b200_process_block_dm_sweep_ex(
                self.h, C.byref(cfg), _ptr(baseband), nbytes, int(on_device), arr, n_dm, res, C.byref(out)))
        else:
            ev = np.zeros(streams * max(max_events, 1), _dtype_of(Event))
            n_ev = (C.c_uint64 * 4)()
            streams = self._ck(self.lib.srtb_b200_process_block_dm_sweep_events(
                self.h, C.byref(cfg), _ptr(baseband), nbytes, int(on_device), arr, n_dm, res, C.byref(out),
                ev.ctypes.data, max_events, n_ev))
        results = [[res[j * streams + s] for s in range(streams)] for j in range(n_dm)]
        nb = max([r.n_boxcars for row in results for r in row] + [0])
        snr = np.array([[list(peaks[j * streams + s].snr)[:nb] for s in range(streams)] for j in range(n_dm)],
                       np.float32).reshape(n_dm, streams, nb)
        idx = np.array([[list(peaks[j * streams + s].peak_index)[:nb] for s in range(streams)] for j in range(n_dm)],
                       np.uint64).reshape(n_dm, streams, nb)
        if max_events is None:
            return results, (snr, idx), [int(best[s]) for s in range(streams)], h_series, list(d_spectrum)
        totals = [int(n_ev[s]) for s in range(streams)]
        events = [ev[s * max_events:s * max_events + min(totals[s], max_events)].copy() for s in range(streams)]
        return results, (snr, idx), [int(best[s]) for s in range(streams)], h_series, list(d_spectrum), events, totals

    def incoherent_dm_search_events(self, d_spectrum, time_count: int, chan_count: int, time_reserved_count: int,
                                    freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms, snr: float,
                                    channel_threshold: float, max_boxcar_length: int, max_events: int,
                                    h_series=None):
        """incoherent_dm_search that also lists every trial's events: returns (results, peaks, best_trial, h_series,
        events, n_events), events a numpy structured array (srtb_b200_event) of the first min(n_events, max_events)"""
        return self.incoherent_dm_search(d_spectrum, time_count, chan_count, time_reserved_count, freq_low, bandwidth,
                                         sample_rate, dm, dms, snr, channel_threshold, max_boxcar_length, h_series,
                                         max_events=max_events)

    def series_events(self, d_series, boxcar_stride: int, trial_stride: int, results, max_events: int):
        """the event pass on caller-owned float32 device series under the headers `results` (DetectResult per
        record): returns (events, n_events), events a numpy structured array of the first min(n_events, max_events)"""
        import numpy as np
        hdr = (DetectResult * len(results))(*results)
        ev = np.zeros(max(max_events, 1), _dtype_of(Event))
        n = C.c_uint64()
        self._ck(self.lib.srtb_b200_series_events(self.h, _ptr(d_series), boxcar_stride, trial_stride, hdr,
                                                  len(results), ev.ctypes.data, max_events, C.byref(n)))
        return ev[:min(n.value, max_events)].copy(), int(n.value)

    def incoherent_dm_search(self, d_spectrum, time_count: int, chan_count: int, time_reserved_count: int,
                             freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms, snr: float,
                             channel_threshold: float, max_boxcar_length: int, h_series=None, max_events=None):
        """semi-coherent DM search of one stream's [chan_count][time_count] complex64 dynamic spectrum (coherently
        dedispersed at dm) over the trial DMs `dms`. Returns (results, (snr, idx), best_trial, h_series): results[d] per
        trial, peaks as numpy arrays [n_dm][n_boxcars] (n_boxcars = the most any trial used), the best trial's index,
        and h_series, a [MAX_BOXCARS][T] float32 array (or the caller's buffer of that size) holding the best trial's
        positive series; T = results[0].time_series_count."""
        import numpy as np
        n_dm = len(dms)
        arr = (C.c_float * n_dm)(*[float(d) for d in dms])
        res = (DetectResult * n_dm)()
        peaks = (Peak * n_dm)()
        best = C.c_int32()
        if h_series is None:
            _, sp, sm = incoherent_shifts(chan_count, freq_low, bandwidth, sample_rate, dm, dms, table=False)
            T = max(time_count - time_reserved_count - sp - sm, 1)
            h_series = np.zeros((MAX_BOXCARS, T), np.float32)
        if max_events is None:
            self._ck(self.lib.srtb_b200_incoherent_dm_search(
                self.h, _ptr(d_spectrum), time_count, chan_count, time_reserved_count, freq_low, bandwidth,
                sample_rate, dm, arr, n_dm, snr, channel_threshold, max_boxcar_length, res, C.cast(peaks, C.c_void_p),
                C.byref(best), _ptr(h_series)))
        else:
            ev = np.zeros(max(max_events, 1), _dtype_of(Event))
            n_ev = C.c_uint64()
            self._ck(self.lib.srtb_b200_incoherent_dm_search_events(
                self.h, _ptr(d_spectrum), time_count, chan_count, time_reserved_count, freq_low, bandwidth,
                sample_rate, dm, arr, n_dm, snr, channel_threshold, max_boxcar_length, res, C.cast(peaks, C.c_void_p),
                C.byref(best), _ptr(h_series), ev.ctypes.data, max_events, C.byref(n_ev)))
        results = [res[d] for d in range(n_dm)]
        nb = max([r.n_boxcars for r in results] + [0])
        snr_a = np.array([list(peaks[d].snr)[:nb] for d in range(n_dm)], np.float32).reshape(n_dm, nb)
        idx_a = np.array([list(peaks[d].peak_index)[:nb] for d in range(n_dm)], np.uint64).reshape(n_dm, nb)
        if max_events is None:
            return results, (snr_a, idx_a), int(best.value), h_series
        return (results, (snr_a, idx_a), int(best.value), h_series, ev[:min(n_ev.value, max_events)].copy(),
                int(n_ev.value))

    def candidate_cutouts(self, d_spectra, time_count: int, chan_count: int, time_reserved_count: int,
                          freq_low: float, bandwidth: float, sample_rate: float, dm: float, requests, width: int,
                          nsub: int, n_rows: int):
        """the frequency-time image and DM-time plane of each request (CutoutRequest, or (center, dm, dm_halfwidth,
        decimation)) on the [chan_count][time_count] complex64 spectra d_spectra (1 to 4 streams, coherently dedispersed
        at dm). Returns numpy float32 arrays (ft [n][nsub][width], dmt [n][n_rows][width], row_dms [n][n_rows])"""
        import numpy as np
        reqs = [r if isinstance(r, CutoutRequest) else CutoutRequest(int(r[0]), float(r[1]), float(r[2]), int(r[3]))
                for r in requests]
        n = len(reqs)
        arr = (CutoutRequest * max(n, 1))(*reqs)
        streams = len(d_spectra)
        sp = (C.c_void_p * max(streams, 1))(*[_ptr(d) for d in d_spectra])
        ft = np.zeros((n, nsub, width), np.float32)
        dmt = np.zeros((n, n_rows, width), np.float32)
        row_dms = np.zeros((n, n_rows), np.float32)
        self._ck(self.lib.srtb_b200_candidate_cutouts(
            self.h, C.cast(sp, C.c_void_p), streams, time_count, chan_count, time_reserved_count, freq_low, bandwidth,
            sample_rate, dm, arr, n, width, nsub, n_rows, ft.ctypes.data, dmt.ctypes.data, row_dms.ctypes.data))
        return ft, dmt, row_dms

    def _submitted(self, cfg: BlockConfig, ticket: int) -> int:
        self._sum_tickets[ticket] = bool(cfg.signal_detect_sum_streams)
        return ticket

    def fold(self, d_spectra, time_count: int, chan_count: int, fold_count: int, phase, nbin: int, nsub: int = 1):
        """fold the first fold_count samples of each [chan_count][time_count] complex64 spectrum in d_spectra (1 to 4
        streams) into nbin phase bins, phase = (phi0, a, b) as fold_phase returns it. Returns numpy arrays (profile
        float64 [streams][nsub][nbin], hits uint64 [nbin], kept uint32 [streams][nsub])"""
        import numpy as np
        streams = len(d_spectra)
        arr = (C.c_void_p * max(streams, 1))(*[_ptr(d) for d in d_spectra])
        profile = np.zeros((streams, nsub, nbin), np.float64)
        hits = np.zeros(nbin, np.uint64)
        kept = np.zeros((streams, nsub), np.uint32)
        phi0, a, b = phase
        self._ck(self.lib.srtb_b200_fold(self.h, arr, streams, time_count, chan_count, fold_count, phi0, a, b, nbin,
                                         nsub, profile.ctypes.data, hits.ctypes.data, kept.ctypes.data))
        return profile, hits, kept

    def fold_coherence(self, d_x, d_y, time_count: int, chan_count: int, fold_count: int, phase, nbin: int,
                       nsub: int = 1):
        """fold the coherence products of two [chan_count][time_count] complex64 spectra X = d_x, Y = d_y (the two
        feeds of one receiver) as fold folds them, over the channels kept in both. Returns numpy arrays (coherence
        float64 [4][nsub][nbin]: AA, BB, CR, CI; hits uint64 [nbin]; kept uint32 [nsub])"""
        import numpy as np
        coherence = np.zeros((4, nsub, nbin), np.float64)
        hits = np.zeros(nbin, np.uint64)
        kept = np.zeros(nsub, np.uint32)
        phi0, a, b = phase
        self._ck(self.lib.srtb_b200_fold_coherence(self.h, _ptr(d_x), _ptr(d_y), time_count, chan_count, fold_count,
                                                   phi0, a, b, nbin, nsub, coherence.ctypes.data, hits.ctypes.data,
                                                   kept.ctypes.data))
        return coherence, hits, kept

    def submit_block(self, cfg: BlockConfig, h_baseband, nbytes: int) -> int:
        """pipelined ingest: H2D on the copy stream overlaps the previous block's compute"""
        return self._submitted(cfg, self._ck(self.lib.srtb_b200_submit_block(self.h, C.byref(cfg), _ptr(h_baseband),
                                                                             nbytes)))

    def submit_block_device(self, cfg: BlockConfig, d_baseband, nbytes: int) -> int:
        return self._submitted(cfg, self._ck(self.lib.srtb_b200_submit_block_device(self.h, C.byref(cfg),
                                                                                    _ptr(d_baseband), nbytes)))

    def _sum_result(self, ticket: int) -> int:
        return 1 if self._sum_tickets.pop(ticket, False) else 0

    def collect_block(self, ticket: int):
        """results per stream, then the sum's when the block was submitted with signal_detect_sum_streams"""
        res = (DetectResult * 5)()
        n = self._ck(self.lib.srtb_b200_collect_block(self.h, ticket, res))
        return [res[i] for i in range(n + self._sum_result(ticket))]

    def submit_block_ex(self, cfg: BlockConfig, baseband, nbytes: int, on_device: bool = False, d_spectrum=None,
                        h_series=None) -> int:
        """ring submission with caller-owned outputs: d_spectrum = per-stream device buffers of N + 2 floats (the
        dynamic spectrum stays there), h_series = pinned host buffer [streams][MAX_BOXCARS][L] for positive series
        ([streams + 1][MAX_BOXCARS][L] with cfg.signal_detect_sum_streams)"""
        out = BlockOutputs()
        for i, t in enumerate(d_spectrum or []):
            out.d_spectrum[i] = _ptr(t)
        out.h_series = _ptr(h_series)
        return self._submitted(cfg, self._ck(self.lib.srtb_b200_submit_block_ex(self.h, C.byref(cfg), _ptr(baseband),
                                                                                nbytes, int(on_device), C.byref(out))))

    def collect_block_ex(self, ticket: int):
        """(results, host pointer of the series buffer, [device pointers of the streams' dynamic spectra]); results end
        with the sum's when the block was submitted with signal_detect_sum_streams"""
        res = (DetectResult * 5)()
        series = C.c_void_p()
        spec = (C.c_void_p * 4)()
        n = self._ck(self.lib.srtb_b200_collect_block_ex(self.h, ticket, res, C.byref(series), spec))
        return [res[i] for i in range(n + self._sum_result(ticket))], series.value, [spec[i] for i in range(n)]

    def submit_block_events(self, cfg: BlockConfig, baseband, nbytes: int, max_events: int, on_device: bool = False,
                            d_spectrum=None, h_series=None) -> int:
        """submit_block_ex that also lists every detector's events (srtb_b200_event), at most max_events per stream
        (and per sum)"""
        out = BlockOutputs()
        for i, t in enumerate(d_spectrum or []):
            out.d_spectrum[i] = _ptr(t)
        out.h_series = _ptr(h_series)
        ticket = self._ck(self.lib.srtb_b200_submit_block_events(self.h, C.byref(cfg), _ptr(baseband), nbytes,
                                                                  int(on_device), C.byref(out), max_events))
        self._event_caps[ticket] = max_events
        return self._submitted(cfg, ticket)

    def collect_block_events(self, ticket: int):
        """collect_block_ex's (results, series pointer, spectra) plus (events, n_events, sum_events, sum_n_events):
        events[s] a numpy structured array (Event's dtype) of stream s's first min(n_events[s], max_events) events, a
        copy of the slot's list; sum_events / sum_n_events the total intensity's (None / 0 without the sum)"""
        import numpy as np
        res = (DetectResult * 5)()
        series = C.c_void_p()
        spec = (C.c_void_p * 4)()
        ev_p = C.c_void_p()
        n_ev = (C.c_uint64 * 5)()
        n = self._ck(self.lib.srtb_b200_collect_block_events(self.h, ticket, res, C.byref(series), spec,
                                                              C.byref(ev_p), n_ev))
        cap = self._event_caps.pop(ticket, 0)
        rows = n + self._sum_result(ticket)
        dt = _dtype_of(Event)
        lists = []
        for r in range(rows):
            k = min(int(n_ev[r]), cap)
            if k:
                buf = (C.c_char * (k * dt.itemsize)).from_address(ev_p.value + r * cap * dt.itemsize)
                lists.append(np.frombuffer(buf, dt, k).copy())
            else:
                lists.append(np.zeros(0, dt))
        totals = [int(n_ev[r]) for r in range(rows)]
        results = [res[i] for i in range(rows)]
        sum_events, sum_total = (lists[n], totals[n]) if rows > n else (None, 0)
        return (results, series.value, [spec[i] for i in range(n)], lists[:n], totals[:n], sum_events, sum_total)

    def debug_set_submit_count(self, value: int):
        self._ck(self.lib.srtb_b200_debug_set_submit_count(self.h, value))

    def block_spectrum_ptr(self, stream: int) -> int:
        return self.lib.srtb_b200_block_spectrum(self.h, stream)

    def sweep_spectrum_ptr(self) -> int:
        """test hook: device pointer of the last trial's dynamic spectrum (last stream) of the latest DM sweep"""
        return self.lib.srtb_b200_sweep_spectrum(self.h)

    def simplify_spectrum(self, d_spectrum, in_width: int, in_height: int, out_width: int, out_height: int,
                          d_intensity, d_pixmap, d_average=None, argb_0: int = GUI_COLOR_0,
                          argb_1: int = GUI_COLOR_1, argb_overflow: int = GUI_COLOR_OVERFLOW):
        """waterfall thumbnail of a [in_height][in_width] complex64 dynamic spectrum (simplify_spectrum_pipe_2):
        d_intensity receives [out_height][out_width] normalised floats, d_pixmap the ARGB32 image, d_average (optional)
        the average intensity before scaling"""
        self._ck(self.lib.srtb_b200_simplify_spectrum(self.h, _ptr(d_spectrum), in_width, in_height, out_width,
                                                      out_height, argb_0, argb_1, argb_overflow, _ptr(d_intensity),
                                                      _ptr(d_pixmap), _ptr(d_average)))

    def cross_spectrum(self, d_a, d_b, count: int, norm: float, d_out):
        """the correlator's cross spectrum: d_out[i] = (norm d_a[i]) conj(d_b[i]), complex64; d_out may be d_a or d_b"""
        self._ck(self.lib.srtb_b200_cross_spectrum(self.h, _ptr(d_a), _ptr(d_b), count, norm, _ptr(d_out)))

    def correlate(self, d_in_1, d_in_2, input_size: int, d_out):
        """the reference's baseband correlator on device bytes: d_out receives input_size // 2 floats, the magnitude of
        the cross-correlation of the two unsigned 8-bit inputs"""
        self._ck(self.lib.srtb_b200_correlate(self.h, _ptr(d_in_1), _ptr(d_in_2), input_size, _ptr(d_out)))

    def correlate_accumulate(self, d_in_1, d_in_2, bits: int, segment_size: int, n_segments: int, d_acc,
                             reset: bool = False):
        """the integrating correlator's accumulation: adds sum_s A_s conj(B_s) over n_segments segments of
        segment_size samples of width bits (1, 2, 4, 8 or -8) of each input into d_acc, segment_size // 2 complex128
        values (16-byte aligned); reset overwrites d_acc instead"""
        self._ck(self.lib.srtb_b200_correlate_accumulate(self.h, _ptr(d_in_1), _ptr(d_in_2), bits, segment_size,
                                                         n_segments, _ptr(d_acc), int(bool(reset))))

    def correlate_finish(self, d_acc, segment_size: int, total_segments: int, d_out):
        """the integrating correlator's result: d_out receives segment_size // 2 floats, the magnitude of the backward
        transform of d_acc scaled by norm / total_segments"""
        self._ck(self.lib.srtb_b200_correlate_finish(self.h, _ptr(d_acc), segment_size, total_segments, _ptr(d_out)))


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


def cluster_events(events, dms, max_candidates: int | None = None):
    """friends-of-friends candidates of an event list (numpy structured array of Event's dtype) searched over the
    trial DMs `dms` (srtb_b200_cluster_events). Returns (candidates, n_candidates): a numpy structured array
    (Candidate's dtype) of the first min(n_candidates, max_candidates) candidates (all when max_candidates is None)"""
    import numpy as np
    lib = load_library()
    ev = np.ascontiguousarray(events, dtype=_dtype_of(Event))
    arr = (C.c_float * max(len(dms), 1))(*[float(d) for d in dms])
    cap = len(ev) if max_candidates is None else max_candidates
    out = np.zeros(max(cap, 1), _dtype_of(Candidate))
    n = C.c_uint64()
    rc = lib.srtb_b200_cluster_events(ev.ctypes.data if len(ev) else None, len(ev), arr, len(dms), out.ctypes.data,
                                      cap, C.byref(n))
    if rc != 0:
        raise SrtbError(rc, lib.srtb_b200_last_error(None).decode())
    return out[:min(n.value, cap)].copy(), int(n.value)


def incoherent_shifts(chan_count: int, freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms,
                      table: bool = True):
    """the incoherent DM search's channel shifts: (s [n_dm][chan_count] int64 numpy array, or None when table is
    False; S+; S-), exactly as srtb_b200_incoherent_dm_search uses them"""
    import numpy as np
    lib = load_library()
    n_dm = len(dms)
    arr = (C.c_float * n_dm)(*[float(d) for d in dms])
    out = np.zeros((n_dm, chan_count), np.int64) if table else None
    sp, sm = C.c_uint64(), C.c_uint64()
    rc = lib.srtb_b200_incoherent_shifts(chan_count, freq_low, bandwidth, sample_rate, dm, arr, n_dm,
                                         None if out is None else out.ctypes.data, C.byref(sp), C.byref(sm))
    if rc < 0:
        raise SrtbError(rc, lib.srtb_b200_last_error(None).decode())
    return out, int(sp.value), int(sm.value)


def incoherent_groups(chan_count: int, freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms):
    """the trial groups srtb_b200_incoherent_dm_search launches with: (order [n_dm], groups [n_groups][2] (first sorted
    slot, count), gspan [n_groups][chan_count][2] (min, max of s + S-), spread), int numpy arrays and an int"""
    import numpy as np
    lib = load_library()
    n_dm = len(dms)
    arr = (C.c_float * n_dm)(*[float(d) for d in dms])
    order = np.zeros(n_dm, np.int32)
    groups = np.zeros((n_dm, 2), np.int32)
    gspan = np.zeros((n_dm, chan_count, 2), np.int32)
    ng, spread = C.c_uint64(), C.c_uint32()
    rc = lib.srtb_b200_incoherent_groups(chan_count, freq_low, bandwidth, sample_rate, dm, arr, n_dm,
                                         order.ctypes.data, groups.ctypes.data, gspan.ctypes.data, C.byref(ng),
                                         C.byref(spread))
    if rc < 0:
        raise SrtbError(rc, lib.srtb_b200_last_error(None).decode())
    return order, groups[:ng.value].copy(), gspan[:ng.value].copy(), int(spread.value)


def fold_phase(period: float, period_derivative: float, sample_rate: float, samples_per_spectrum_sample: int,
               first_sample: int):
    """(phi0, a, b) of the fold's phase model for a block starting at baseband sample first_sample, exactly as
    srtb_b200_fold_phase computes them: phi_j = phi0 + a j + b j^2 at spectrum sample j"""
    lib = load_library()
    phi0, a, b = C.c_double(), C.c_double(), C.c_double()
    rc = lib.srtb_b200_fold_phase(period, period_derivative, sample_rate, samples_per_spectrum_sample, first_sample,
                                  C.byref(phi0), C.byref(a), C.byref(b))
    if rc < 0:
        raise SrtbError(rc, lib.srtb_b200_last_error(None).decode())
    return phi0.value, a.value, b.value
