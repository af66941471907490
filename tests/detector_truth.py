"""Float64 truth of the single-pulse detector (signal_detect_pipe_2, restated in oracle/srtb_oracle.cpp), with a
first-order worst-case bound on what the GPU's fp32 / fp64 operation order can leave in every output.

Test infrastructure only: numpy on the host, no GPU. A caller holding the spectrum on a GPU may form the column sums
there (in float64) and pass them to truth_from_columns.

Rounding bounds, u = 2^-24 (unit roundoff of fp32), d = exact mean-removed series, A = exact column sums:

  row 0   e0[j] = (C+1) u (A[j] + mean(A)) + 3u mean(A) + u |d[j]|
          - every |y|^2 is x*x + y*y in fp32 (one product and one add or fma: <= 2u |y|^2), and the C powers of a
            column are added in fp32 in whatever order a route uses: C - 1 additions of non-negative terms, each
            rounding at most u times the column total. Together (C+1) u A[j]; additions of zeros are exact.
          - the mean is an fp64 sum of those fp32 sums (it inherits (C+1) u mean(A)), rounded to fp32 once (u) and
            divided by float(ts_count) in fp32 (u): 2u mean(A), written as 3u to keep the fp64 sum's rounding covered.
          - d = ts - mean in fp32: u |d[j]|.
  boxcar  e_b[i] = sum_{k=i+1..i+b} e0[k] + u (|acc[i+b]| + |acc[i]|) + u |S_b[i]| + n 2^-53 max|acc|
          the scan runs in fp64 over the fp32 values of row 0; a difference of two prefixes only sees the errors of
          the window. Each prefix is rounded to fp32 once (u |acc|), the difference is taken in fp32 (u |S|), and the
          fp64 scan itself rounds at most n times 2^-53 of its largest prefix.
  var     var = sum S^2 / n. The GPU sums the squares of its fp32 series in fp64 and divides in fp32:
          e_var = E / n + 3u (var + E / n),  E = sum (2 |S| e + e^2) + n 2^-53 sum S^2
          (one rounding of the fp64 sum to fp32, one of the division, one spare for the fp64 sum's own order).
  thr     thr = snr * sqrtf(var): snr is the fp32 value the caller passed; sqrtf and the product round once each.
          thr lies in snr [sqrt(max(var - e_var, 0)), sqrt(var + e_var)] (1 -/+ 2u); e_thr is the larger distance.
  count   the GPU count lies in [#(S > thr + m), #(S >= thr - m)], m = e_b[i] + e_thr.

Exact fields: zero_count, time_series_count, detect_enabled, n_boxcars, boxcar_length, series_length.
detect_enabled is the reference's fp32 expression float(zc) < float(chan_thr) * float(C).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

U = 2.0 ** -24
U64 = 2.0 ** -53
MAX_BOXCARS = 32


def ts_count_for(time_count: int, reserved: int) -> int:
    """the reference's trimming rule: a reservation of the whole row (or more) keeps the whole row"""
    return time_count if time_count <= reserved else time_count - reserved


def detect_enabled(zero_count: int, chan_count: int, chan_thr: float) -> bool:
    return bool(np.float32(zero_count) < np.float32(chan_thr) * np.float32(chan_count))


def boxcar_lengths(ts_count: int, max_boxcar: int) -> list[int]:
    """1, then 2, 4, .. while b <= max_boxcar and b < ts_count, at most 32 in all"""
    out = [1]
    b = 2
    while b <= max_boxcar and b < ts_count and len(out) < MAX_BOXCARS:
        out.append(b)
        b *= 2
    return out


@dataclass
class Truth:
    zero_count: int
    time_series_count: int
    detect_enabled: bool
    n_boxcars: int
    chan_count: int
    boxcar_length: list = field(default_factory=list)
    series_length: list = field(default_factory=list)
    series: list = field(default_factory=list)       # float64 [n_b] per boxcar; series[0] also when disabled
    err: list = field(default_factory=list)          # bound of |gpu - truth| per element, same shapes
    variance: list = field(default_factory=list)
    var_err: list = field(default_factory=list)
    threshold: list = field(default_factory=list)
    thr_err: list = field(default_factory=list)
    count_lo: list = field(default_factory=list)
    count_hi: list = field(default_factory=list)


def zero_count(first: np.ndarray) -> int:
    """masked channels: |y|^2 == 0 evaluated in fp32, as the reference does (a subnormal square counts as zero)"""
    y = np.asarray(first, np.complex64)
    return int(np.count_nonzero(y.real * y.real + y.imag * y.imag == np.float32(0)))


def column_power(spec: np.ndarray, ts_count: int) -> tuple[np.ndarray, int]:
    """[C][L] complex64 -> (A[j] = sum_c |y[c, j]|^2 over j < ts_count in float64, zero count of the first samples)"""
    y = np.asarray(spec)
    p = y[:, :ts_count].real.astype(np.float64) ** 2 + y[:, :ts_count].imag.astype(np.float64) ** 2
    return p.sum(axis=0), zero_count(y[:, 0])


def truth_from_columns(A, chan_count: int, zero_count: int, snr: float, chan_thr: float, max_boxcar: int,
                       fp32_oracle: bool = False) -> Truth:
    """A: exact column sums (float64, ts_count of them), each a sum of chan_count powers.
    fp32_oracle: widen the bounds for the CPU oracle's operation order instead of the GPU's: its mean and its sum of
    squares are pairwise fp32 sums (ceil(log2 n) + 1 roundings deep), and its scan is serial fp32, so every prefix
    carries u times the sum of the magnitudes of all prefixes up to it."""
    A = np.asarray(A, dtype=np.float64)
    n0 = A.size
    C = chan_count
    mean_a = A.mean()
    d = A - mean_a
    e0 = (C + 1) * U * (A + mean_a) + 3 * U * mean_a + U * np.abs(d)
    if fp32_oracle:
        e0 = e0 + (np.ceil(np.log2(max(n0, 2))) + 1) * U * mean_a
    en = detect_enabled(zero_count, C, chan_thr)
    t = Truth(zero_count=zero_count, time_series_count=n0, detect_enabled=en, n_boxcars=0, chan_count=C)
    t.series.append(d)
    t.err.append(e0)
    if not en:
        return t
    acc = np.cumsum(d)
    cum_e0 = np.concatenate([[0.0], np.cumsum(e0)])   # cum_e0[k] = sum e0[:k]
    scan_err = n0 * U64 * np.abs(acc).max()
    if fp32_oracle:
        scan_err = scan_err + U * np.cumsum(np.abs(acc))
    snr32 = float(np.float32(snr))
    for b in boxcar_lengths(n0, max_boxcar):
        if b == 1:
            S, e = d, e0
        else:
            n = n0 - b
            S = acc[b:] - acc[:n]
            se = scan_err if np.isscalar(scan_err) else scan_err[b:] + scan_err[:n]
            e = (cum_e0[b + 1:n0 + 1] - cum_e0[1:n + 1]) + U * (np.abs(acc[b:]) + np.abs(acc[:n])) + U * np.abs(S) + se
            t.series.append(S)
            t.err.append(e)
        n = S.size
        var = float(np.dot(S, S) / n)
        E = float(np.sum(2 * np.abs(S) * e + e * e)) + n * U64 * float(np.dot(S, S))
        var_err = E / n + 3 * U * (var + E / n)
        if fp32_oracle:
            var_err += (np.ceil(np.log2(max(n, 2))) + 1) * U * (var + E / n)
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


def signal_detect(spec: np.ndarray, time_count: int, chan_count: int, reserved: int, snr: float, chan_thr: float,
                  max_boxcar: int, **kw) -> Truth:
    """per-pipe detector on a [C][L] spectrum (zero count over the first sample of every channel)"""
    y = np.asarray(spec).reshape(chan_count, time_count)
    A, zc = column_power(y, ts_count_for(time_count, reserved))
    return truth_from_columns(A, chan_count, zc, snr, chan_thr, max_boxcar, **kw)


def signal_detect_v1(spec: np.ndarray, count_per_batch: int, batch_size: int, snr: float, chan_thr: float,
                     max_boxcar: int, **kw) -> Truth:
    """v1 detector on a [time][frequency] spectrum AFTER its SK v1: one value per spectrum (sum over frequency),
    nothing trimmed, zero count over the first spectrum"""
    y = np.asarray(spec).reshape(batch_size, count_per_batch)
    A, _ = column_power(y.T, batch_size)
    return truth_from_columns(A, count_per_batch, zero_count(y[0]), snr, chan_thr, max_boxcar, **kw)


def compare(got, got_series, truth: Truth, rows=None) -> dict:
    """check a detect result header (srtb_b200.DetectResult or oracle_lib.DetectResult) and, when given, its series
    rows [MAX_BOXCARS][>= n] against the truth. Returns the largest error / bound of the series, the variance and the
    threshold. Raises AssertionError on the first violation. rows: the series rows to check (default every boxcar's)."""
    assert int(got.zero_count) == truth.zero_count, (int(got.zero_count), truth.zero_count)
    assert int(got.time_series_count) == truth.time_series_count
    assert bool(got.detect_enabled) == truth.detect_enabled
    assert int(got.n_boxcars) == truth.n_boxcars, (int(got.n_boxcars), truth.n_boxcars)
    worst = {"series": 0.0, "variance": 0.0, "threshold": 0.0}

    def ratio(err, bound):
        err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
        assert np.all(np.isfinite(err))
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
        return float(r.max()) if r.size else 0.0

    for b in range(truth.n_boxcars):
        assert int(got.boxcar_length[b]) == truth.boxcar_length[b]
        assert int(got.series_length[b]) == truth.series_length[b]
        rv = ratio(abs(float(got.variance[b]) - truth.variance[b]), truth.var_err[b])
        rt = ratio(abs(float(got.threshold[b]) - truth.threshold[b]), truth.thr_err[b])
        assert rv <= 1, f"boxcar {b}: variance {got.variance[b]} vs {truth.variance[b]} (bound {truth.var_err[b]:.3e})"
        assert rt <= 1, f"boxcar {b}: threshold {got.threshold[b]} vs {truth.threshold[b]} (bound {truth.thr_err[b]:.3e})"
        c = int(got.signal_count[b])
        assert truth.count_lo[b] <= c <= truth.count_hi[b], \
            f"boxcar {b}: count {c} outside [{truth.count_lo[b]}, {truth.count_hi[b]}]"
        worst["variance"] = max(worst["variance"], rv)
        worst["threshold"] = max(worst["threshold"], rt)
    if got_series is not None:
        for b in (range(truth.n_boxcars) if rows is None else rows):
            n = truth.series_length[b] if b < truth.n_boxcars else truth.time_series_count
            r = ratio(np.abs(np.asarray(got_series[b][:n], np.float64) - truth.series[b]), truth.err[b])
            assert r <= 1, f"boxcar {b}: series outside its bound by {r:.3g}x"
            worst["series"] = max(worst["series"], r)
    return worst
