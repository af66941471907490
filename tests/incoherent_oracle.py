"""Float64 restatement of the semi-coherent DM search (srtb_b200_incoherent_dm_search), for the tests.

For trial DMs near the coherent `dm`, each channel c of the [C][L] dynamic spectrum is shifted by the residual
dispersive delay between channels, rounded to whole samples of dt = 2C / sample_rate:

    f_ref = float32(freq_low + bandwidth)            (the chirp's f_c: top edge for bandwidth > 0, bottom for < 0)
    f(c)  = freq_low + bandwidth (c + 0.5) / C
    s[d][c] = round_half_away(4.148808e3 (DM_d - dm) (1/f(c)^2 - 1/f_ref^2) sample_rate / (2C))
    S+ = max(0, max s), S- = max(0, -min s), T = ts - S+ - S-
    v_d[j] = sum_c |x[c][j + S- + s[d][c]]|^2,  j < T

and every v_d goes through signal_detect_pipe_2's detector (mean removal, boxcars 1, 2, 4, ..., variance, threshold,
count) with per-boxcar peaks (max / sqrt(variance), first index of the maximum). The shift arithmetic is the library's
double-precision expression in the same order, so the tables agree exactly, half-sample ties included.
"""
from __future__ import annotations

import numpy as np

from detector_truth import boxcar_lengths, detect_enabled

DISPERSION_CONSTANT = 4.148808e3
MAX_BOXCARS = 32


def shift_values(chan_count: int, freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms) -> np.ndarray:
    """the unrounded shifts [n_dm][C] in float64, in the library's order of operations"""
    fl, bw, sr = (float(np.float32(v)) for v in (freq_low, bandwidth, sample_rate))
    f_ref = float(np.float32(np.float32(freq_low) + np.float32(bandwidth)))
    scale = sr / (2.0 * chan_count)
    c = np.arange(chan_count, dtype=np.float64)
    f = fl + bw * (c + 0.5) / chan_count
    k = (1.0 / (f * f) - 1.0 / (f_ref * f_ref)) * scale * DISPERSION_CONSTANT
    ddm = np.asarray([float(np.float32(d)) for d in dms], np.float64) - float(np.float32(dm))
    return ddm[:, None] * k[None, :]


def round_half_away(v: np.ndarray) -> np.ndarray:
    """llround: halves go away from zero"""
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)


def shifts(chan_count: int, freq_low: float, bandwidth: float, sample_rate: float, dm: float, dms):
    """(s [n_dm][C] int64, S+, S-)"""
    s = round_half_away(shift_values(chan_count, freq_low, bandwidth, sample_rate, dm, dms))
    return s, int(max(0, s.max())), int(max(0, -s.min()))


def series(power: np.ndarray, ts_count: int, s: np.ndarray, s_plus: int, s_minus: int) -> np.ndarray:
    """v [n_dm][T] in float64 from the power |x|^2 [C][L]"""
    T = ts_count - s_plus - s_minus
    C = power.shape[0]
    out = np.zeros((s.shape[0], T), np.float64)
    for d in range(s.shape[0]):
        for c in range(C):
            o = s_minus + int(s[d, c])
            out[d] += power[c, o:o + T]
    return out


def detect(v: np.ndarray, zero_count: int, chan_count: int, snr: float, chan_thr: float, max_boxcar: int) -> dict:
    """signal_detect_pipe_2 on one series v (float64), with the peaks of every boxcar series"""
    T = len(v)
    out = {"zero_count": zero_count, "time_series_count": T, "detect_enabled": detect_enabled(zero_count, chan_count,
                                                                                              chan_thr),
           "boxcar_length": [], "series_length": [], "variance": [], "threshold": [], "signal_count": [],
           "peak_snr": [], "peak_index": [], "series": [], "margin": []}
    if not out["detect_enabled"]:
        out["n_boxcars"] = 0
        return out
    d = v - v.sum() / T
    acc = np.cumsum(d)
    for b in boxcar_lengths(T, max_boxcar):
        sb = d if b == 1 else acc[b:] - acc[:T - b]
        var = float(np.mean(sb * sb))
        thr = float(snr) * np.sqrt(var)
        out["boxcar_length"].append(b)
        out["series_length"].append(len(sb))
        out["variance"].append(var)
        out["threshold"].append(thr)
        out["signal_count"].append(int(np.count_nonzero(sb > thr)))
        out["margin"].append(float(np.min(np.abs(sb - thr))) if thr > 0 else 0.0)
        out["peak_snr"].append(float(sb.max() / np.sqrt(var)) if var > 0 else 0.0)
        out["peak_index"].append(int(np.argmax(sb)))
        out["series"].append(sb)
    out["n_boxcars"] = len(out["boxcar_length"])
    return out


def search(spec: np.ndarray, time_reserved_count: int, freq_low: float, bandwidth: float, sample_rate: float,
           dm: float, dms, snr: float, chan_thr: float, max_boxcar: int):
    """the whole search on a complex [C][L] spectrum: (per-trial detect() dicts, best trial, (s, S+, S-))"""
    C, L = spec.shape
    s, sp, sm = shifts(C, freq_low, bandwidth, sample_rate, dm, dms)
    power = np.abs(spec.astype(np.complex128)) ** 2
    zc = int(np.count_nonzero(power[:, 0] == 0))
    v = series(power, L - time_reserved_count, s, sp, sm)
    trials = [detect(v[d], zc, C, snr, chan_thr, max_boxcar) for d in range(len(dms))]
    return trials, best_trial(trials), (s, sp, sm)


def best_trial(trials) -> int:
    """positive trials first, then the largest peak S/N over the boxcars, then the lowest index"""
    best, best_pos, best_snr = -1, False, 0.0
    for j, t in enumerate(trials):
        if not t["detect_enabled"]:
            continue
        pos = any(c > 0 for c in t["signal_count"])
        snr = max(t["peak_snr"], default=-np.inf)
        if best < 0 or (pos and not best_pos) or (pos == best_pos and snr > best_snr):
            best, best_pos, best_snr = j, pos, snr
    return max(best, 0)
