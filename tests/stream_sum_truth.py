"""Float64 truth of the total-intensity detector (signal_detect_sum_streams, csrc/stream_sum.cuh) with a first-order bound
of what its fp32 operation order can leave, in the form of tests/detector_truth.py.

Test infrastructure only (numpy on the host; the column powers may be formed on a GPU in float64 and passed in).

The sum's series before mean removal, S streams, C channels, M (mismatched channel, keeping stream) pairs, u = 2^-24:
  v[j] = sum_s R_s[j] - sum over the M pairs of |x_s[c][j]|^2,   R_s = the stream's own fp32 column sum
  - R_s[j] carries (C + 1) u R_s[j] (detector_truth: C - 1 fp32 additions of non-negative powers, 2u per power);
  - the S - 1 additions of the R_s round at most u times the running total each, which is at most T[j] = sum_s R_s[j]
    (the exact sums of every stream over all channels, removed rows included);
  - each of the M removed powers carries 2u of itself, and each subtraction rounds at most u times the running value,
    which never exceeds T[j]: 3u T[j] per pair.
  So e_v[j] = (C + S + 3M) u T[j]. A strong row removed from the sum keeps its rounding in the bound through T.
  Mean removal, scan, boxcars, variance, threshold and counts then follow detector_truth.truth_from_columns, whose
  row-0 bound (C + 1) u (A + mean A) + 3u mean A + u |d| becomes e_v + mean(e_v) + 3u mean A + u |d|.
"""
from __future__ import annotations

import numpy as np

from detector_truth import MAX_BOXCARS, U, U64, Truth, boxcar_lengths, detect_enabled  # noqa: F401


def sum_truth(A, T, chan_count: int, streams: int, pairs: int, zero_count: int, snr: float, chan_thr: float,
              max_boxcar: int) -> Truth:
    """A: exact summed power over the kept channels (float64, ts_count values); T: exact sum of every stream's column
    sums over all channels; pairs: the number of (mismatched channel, keeping stream) pairs"""
    A = np.asarray(A, np.float64)
    T = np.asarray(T, np.float64)
    n0 = A.size
    mean_a = A.mean()
    d = A - mean_a
    ev = (chan_count + streams + 3 * pairs) * U * T
    e0 = ev + ev.mean() + 3 * U * mean_a + U * np.abs(d)
    en = detect_enabled(zero_count, chan_count, chan_thr)
    t = Truth(zero_count=zero_count, time_series_count=n0, detect_enabled=en, n_boxcars=0, chan_count=chan_count)
    t.series.append(d)
    t.err.append(e0)
    if not en:
        return t
    acc = np.cumsum(d)
    cum_e0 = np.concatenate([[0.0], np.cumsum(e0)])
    scan_err = n0 * U64 * np.abs(acc).max()
    snr32 = float(np.float32(snr))
    for b in boxcar_lengths(n0, max_boxcar):
        if b == 1:
            S, e = d, e0
        else:
            n = n0 - b
            S = acc[b:] - acc[:n]
            e = (cum_e0[b + 1:n0 + 1] - cum_e0[1:n + 1]) + U * (np.abs(acc[b:]) + np.abs(acc[:n])) + U * np.abs(S) \
                + scan_err
            t.series.append(S)
            t.err.append(e)
        n = S.size
        var = float(np.dot(S, S) / n)
        E = float(np.sum(2 * np.abs(S) * e + e * e)) + n * U64 * float(np.dot(S, S))
        var_err = E / n + 3 * U * (var + E / n)
        thr = snr32 * np.sqrt(var)
        hi = snr32 * np.sqrt(var + var_err) * (1 + 2 * U)
        lo = snr32 * np.sqrt(max(var - var_err, 0.0)) * (1 - 2 * U)
        thr_err = max(hi - thr, thr - lo)
        m = e + thr_err
        t.boxcar_length.append(b)
        t.series_length.append(n)
        t.variance.append(var)
        t.var_err.append(var_err)
        t.threshold.append(thr)
        t.thr_err.append(thr_err)
        t.count_lo.append(int(np.count_nonzero(S > thr + m)))
        t.count_hi.append(int(np.count_nonzero(S >= thr - m)))
    t.n_boxcars = len(t.boxcar_length)
    return t
