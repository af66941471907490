"""ctypes access to the CPU oracle (oracle/libsrtb_oracle.so) — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module; the product path never does.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE_DIR = ROOT / "oracle"
LIB = ORACLE_DIR / "libsrtb_oracle.so"
MAXB = 32


class DetectResult(C.Structure):
    _fields_ = [
        ("zero_count", C.c_uint64),
        ("time_series_count", C.c_uint64),
        ("detect_enabled", C.c_int32),
        ("n_boxcars", C.c_int32),
        ("boxcar_length", C.c_uint64 * MAXB),
        ("series_length", C.c_uint64 * MAXB),
        ("signal_count", C.c_uint64 * MAXB),
        ("variance", C.c_float * MAXB),
        ("threshold", C.c_float * MAXB),
    ]


class ChainConfig(C.Structure):
    _fields_ = [
        ("baseband_input_count", C.c_uint64),
        ("baseband_input_bits", C.c_int32),
        ("window", C.c_int32),
        ("baseband_freq_low", C.c_float),
        ("baseband_bandwidth", C.c_float),
        ("baseband_sample_rate", C.c_float),
        ("dm", C.c_float),
        ("baseband_reserve_sample", C.c_int32),
        ("rfi_average_threshold", C.c_float),
        ("rfi_sk_threshold", C.c_float),
        ("spectrum_channel_count", C.c_uint64),
        ("snr_threshold", C.c_float),
        ("channel_threshold", C.c_float),
        ("max_boxcar_length", C.c_uint64),
        ("rfi_pairs", C.POINTER(C.c_float)),
        ("n_rfi_pairs", C.c_uint64),
    ]


def build():
    if not LIB.exists() or LIB.stat().st_mtime < (ORACLE_DIR / "srtb_oracle.cpp").stat().st_mtime:
        subprocess.run(["make", "-C", str(ORACLE_DIR), "libsrtb_oracle.so"], check=True,
                       capture_output=True)


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a


class Oracle:
    def __init__(self):
        build()
        self.lib = C.CDLL(str(LIB))
        L = self.lib
        P, SZ, F, I = C.c_void_p, C.c_size_t, C.c_float, C.c_int
        L.srtb_oracle_window.restype = F
        L.srtb_oracle_window.argtypes = [I, SZ, SZ]
        L.srtb_oracle_unpack.argtypes = [P, SZ, I, I, P]
        L.srtb_oracle_unpack_interleaved_2.argtypes = [P, SZ, I, I, P, P]
        L.srtb_oracle_unpack_snap1.argtypes = [P, SZ, I, P, P]
        L.srtb_oracle_unpack_gznupsr_a1.argtypes = [P, SZ, I, I, C.POINTER(P)]
        L.srtb_oracle_fft_c2c.argtypes = [P, SZ, I]
        L.srtb_oracle_fft_r2c.argtypes = [P, SZ]
        L.srtb_oracle_watfft.argtypes = [P, SZ, SZ]
        L.srtb_oracle_norm_coefficient.restype = F
        L.srtb_oracle_norm_coefficient.argtypes = [SZ, SZ]
        L.srtb_oracle_rfi_s1_average.argtypes = [P, SZ, F, SZ, P, P]
        L.srtb_oracle_eval_rfi_ranges.restype = SZ
        L.srtb_oracle_eval_rfi_ranges.argtypes = [C.c_char_p, P, SZ]
        L.srtb_oracle_rfi_range_to_bins.argtypes = [F, F, F, F, SZ, C.POINTER(SZ), C.POINTER(SZ)]
        L.srtb_oracle_rfi_manual.restype = SZ
        L.srtb_oracle_rfi_manual.argtypes = [P, SZ, F, F, P, SZ]
        L.srtb_oracle_dedisperse.argtypes = [P, SZ, F, F, F, F]
        L.srtb_oracle_nsamps_reserved.restype = SZ
        L.srtb_oracle_nsamps_reserved.argtypes = [SZ, SZ, F, F, F, F, I]
        L.srtb_oracle_sk_thresholds.argtypes = [SZ, F, P, P]
        L.srtb_oracle_rfi_s2.argtypes = [P, SZ, SZ, F, P, P]
        L.srtb_oracle_signal_detect.argtypes = [P, SZ, SZ, SZ, F, F, SZ, C.POINTER(DetectResult), P]
        L.srtb_oracle_chain.argtypes = [P, C.POINTER(ChainConfig), P, C.POINTER(DetectResult), P, P]
        L.srtb_oracle_num_threads.restype = I
        L.srtb_oracle_count_signal.restype = C.c_uint64
        L.srtb_oracle_count_signal.argtypes = [P, SZ, F]

    # ---- unpack
    def window(self, window, i, n):
        return float(self.lib.srtb_oracle_window(window, i, n))

    def unpack(self, raw: np.ndarray, out_count: int, bits: int, window: int = 0):
        raw = np.ascontiguousarray(raw)
        out = np.empty(out_count, np.float32)
        rc = self.lib.srtb_oracle_unpack(raw.ctypes.data, out_count, bits, window, out.ctypes.data)
        if rc != 0:
            raise ValueError(f"unsupported bits {bits}")
        return out

    def unpack_interleaved_2(self, raw, out_count, bits, window=0):
        raw = np.ascontiguousarray(raw)
        o1, o2 = np.empty(out_count, np.float32), np.empty(out_count, np.float32)
        rc = self.lib.srtb_oracle_unpack_interleaved_2(raw.ctypes.data, out_count, bits, window,
                                                       o1.ctypes.data, o2.ctypes.data)
        if rc != 0:
            raise ValueError(f"unsupported bits {bits}")
        return o1, o2

    def unpack_snap1(self, raw, out_count, window=0):
        raw = np.ascontiguousarray(raw)
        o1, o2 = np.zeros(out_count, np.float32), np.zeros(out_count, np.float32)
        self.lib.srtb_oracle_unpack_snap1(raw.ctypes.data, out_count, window, o1.ctypes.data, o2.ctypes.data)
        return o1, o2

    def unpack_gznupsr_a1(self, raw, out_count, streams, window=0):
        raw = np.ascontiguousarray(raw)
        outs = [np.zeros(out_count, np.float32) for _ in range(streams)]
        arr = (C.c_void_p * streams)(*[o.ctypes.data for o in outs])
        rc = self.lib.srtb_oracle_unpack_gznupsr_a1(raw.ctypes.data, out_count, streams, window, arr)
        assert rc == 0
        return outs

    # ---- FFT (restated naive radix-2, f32)
    def fft_c2c(self, x: np.ndarray, direction: int):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        self.lib.srtb_oracle_fft_c2c(y.ctypes.data, y.size, direction)
        return y

    def fft_r2c(self, x: np.ndarray):
        n = x.size
        buf = np.zeros(n + 2, np.float32)
        buf[:n] = x
        self.lib.srtb_oracle_fft_r2c(buf.ctypes.data, n)
        return buf.view(np.complex64).copy()  # n/2 + 1 bins

    def watfft(self, x: np.ndarray, length: int, batch: int):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        self.lib.srtb_oracle_watfft(y.ctypes.data, length, batch)
        return y

    # ---- RFI stage 1
    def norm_coefficient(self, in_count, channel_count):
        return float(self.lib.srtb_oracle_norm_coefficient(in_count, channel_count))

    def rfi_s1_average(self, x, threshold, channel_count):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        mean = C.c_float()
        mask = np.zeros(y.size, np.uint8)
        self.lib.srtb_oracle_rfi_s1_average(y.ctypes.data, y.size, threshold, channel_count,
                                            C.addressof(mean), mask.ctypes.data)
        return y, float(mean.value), mask

    def eval_rfi_ranges(self, s: str):
        buf = np.zeros(128, np.float32)
        n = self.lib.srtb_oracle_eval_rfi_ranges(s.encode(), buf.ctypes.data, 64)
        return [(float(buf[2 * i]), float(buf[2 * i + 1])) for i in range(min(n, 64))]

    def rfi_range_to_bins(self, f1, f2, freq_low, bandwidth, in_count):
        lo, hi = C.c_size_t(), C.c_size_t()
        ok = self.lib.srtb_oracle_rfi_range_to_bins(f1, f2, freq_low, bandwidth, in_count,
                                                    C.byref(lo), C.byref(hi))
        return (lo.value, hi.value) if ok else None

    def rfi_manual(self, x, freq_low, bandwidth, pairs):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        p = np.asarray(pairs, np.float32).reshape(-1)
        self.lib.srtb_oracle_rfi_manual(y.ctypes.data, y.size, freq_low, bandwidth, p.ctypes.data, p.size // 2)
        return y

    # ---- dedisperse
    def dedisperse(self, x, f_min, f_c, df, dm):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        self.lib.srtb_oracle_dedisperse(y.ctypes.data, y.size, f_min, f_c, df, dm)
        return y

    def nsamps_reserved(self, n, c, freq_low, bw, fs, dm, reserve):
        return int(self.lib.srtb_oracle_nsamps_reserved(n, c, freq_low, bw, fs, dm, int(reserve)))

    # ---- SK
    def sk_thresholds(self, time_count, thr):
        lo, hi = C.c_float(), C.c_float()
        self.lib.srtb_oracle_sk_thresholds(time_count, thr, C.addressof(lo), C.addressof(hi))
        return float(lo.value), float(hi.value)

    def rfi_s2(self, x, time_count, chan_count, thr):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        sk = np.zeros(chan_count, np.float32)
        zap = np.zeros(chan_count, np.uint8)
        self.lib.srtb_oracle_rfi_s2(y.ctypes.data, time_count, chan_count, thr, sk.ctypes.data, zap.ctypes.data)
        return y, sk, zap

    # ---- detect
    def signal_detect(self, x, time_count, chan_count, reserved, snr, chan_thr, max_boxcar):
        x = np.ascontiguousarray(x, dtype=np.complex64)
        res = DetectResult()
        series = np.zeros((MAXB, time_count), np.float32)
        self.lib.srtb_oracle_signal_detect(x.ctypes.data, time_count, chan_count, reserved, snr, chan_thr,
                                           max_boxcar, C.byref(res), series.ctypes.data)
        return res, series

    # ---- alternates of the refft path ([time][frequency])
    def sk_v1(self, x, fft_bins, time_counts, thr):
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        sk = np.zeros(fft_bins, np.float32)
        zap = np.zeros(fft_bins, np.uint8)
        self.lib.srtb_oracle_sk_v1(C.c_void_p(y.ctypes.data), C.c_size_t(fft_bins), C.c_size_t(time_counts), C.c_float(thr),
                                   C.c_void_p(sk.ctypes.data), C.c_void_p(zap.ctypes.data))
        return y, sk, zap

    def signal_detect_v1(self, x, count_per_batch, batch_size, sk_thr, snr, chan_thr, max_boxcar):
        """returns (spectrum after SK v1, result header, series [MAXB][batch_size])"""
        y = np.ascontiguousarray(x, dtype=np.complex64).copy()
        res = DetectResult()
        series = np.zeros((MAXB, batch_size), np.float32)
        self.lib.srtb_oracle_signal_detect_v1(C.c_void_p(y.ctypes.data), C.c_size_t(count_per_batch), C.c_size_t(batch_size),
                                              C.c_float(sk_thr), C.c_float(snr), C.c_float(chan_thr),
                                              C.c_size_t(max_boxcar), C.byref(res), C.c_void_p(series.ctypes.data))
        return y, res, series

    # ---- whole chain (CPU baseline)
    def chain(self, baseband: np.ndarray, cfg: ChainConfig):
        n = int(cfg.baseband_input_count)
        work = np.zeros(n + 2, np.float32)
        res = DetectResult()
        nc = n // 2
        batch = min(int(cfg.spectrum_channel_count), nc)
        L = nc // batch
        series = np.zeros((MAXB, L), np.float32)
        stage_s = np.zeros(7, np.float64)
        baseband = np.ascontiguousarray(baseband)
        rc = self.lib.srtb_oracle_chain(baseband.ctypes.data, C.byref(cfg), work.ctypes.data, C.byref(res),
                                        series.ctypes.data, stage_s.ctypes.data)
        assert rc == 0
        return work, res, series, stage_s

    def count_signal(self, v, snr):
        v = np.ascontiguousarray(v, dtype=np.float32)
        return int(self.lib.srtb_oracle_count_signal(v.ctypes.data, v.size, snr))

    def set_threads(self, n: int):
        self.lib.srtb_oracle_set_threads(int(n))

    def num_threads(self):
        return int(self.lib.srtb_oracle_num_threads())


_inst = None


def load() -> Oracle:
    global _inst
    if _inst is None:
        _inst = Oracle()
    return _inst
