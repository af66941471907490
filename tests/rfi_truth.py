"""Float64 truth of the RFI zap decisions a block makes before the detector sees it, and a host mirror of which kernels
make them. No GPU needed: the functions take numpy arrays, or torch tensors (on any device) where noted, so that the
GPU tests can form the truth of long blocks on the device.

Three decisions: s1 zaps bin k when |X_k|^2 > avg_thr * mean(|X|^2) (the mean over bins 0 .. Nc - 1, before the manual
ranges are zeroed); the manual ranges zero their bins whatever their power; SK zaps a channel row whose spectral
kurtosis L * sum p^2 / (sum p)^2 over its L time samples lies outside the scaled window of sk_bounds. A decision whose
statistic lies within a relative `margin` of its edge may go either way in fp32; compare_decisions reports the others.
"""
from dataclasses import dataclass

import numpy as np

ROW16 = (1 << 10, 1 << 11, 1 << 12)          # sixteen-point row kernel, s1 + chirp on load, SK in its epilogue
BIGROW = (1 << 13, 1 << 14)                  # whole-row kernel, the same
LONG = tuple(1 << q for q in range(15, 19))  # column sweep with s1 + chirp on load, SK from per-tile statistics
MEAN_ROUTES = ("post", "fixup2", "fixup3", "fixup4", "rows_split")
TAIL_ROUTES = ("row16", "row8_512", "bigrow", "long", "unfused")

SIMPLE, INTERLEAVED_2, NAOCPSR_SNAP1, GZNUPSR_A1_2, GZNUPSR_A1_4 = range(5)   # srtb_b200.FORMAT_*
STREAMS = {SIMPLE: 1, INTERLEAVED_2: 2, NAOCPSR_SNAP1: 2, GZNUPSR_A1_2: 2, GZNUPSR_A1_4: 4}


# ----------------------------------------------------------------------------------------------------- route mirror
def _plan3(q):
    """srtb_b200.cu plan3 (lines 697-704): the three-sweep factorisation, last factor <= 8 where possible"""
    l1 = (q + 2) // 3
    big = (q - l1 + 1) // 2
    small = q - l1 - big
    return (l1, small, big) if big <= 8 else (l1, big, small)


def _plan4(q):
    """srtb_b200.cu plan4 (lines 709-715): four sweeps for 2^27 .. 2^30 points"""
    l3 = 8 if q >= 29 else 7
    r = q - l3
    l0 = (r + 2) // 3
    l1 = (r - l0 + 1) // 2
    return l0, l1, r - l0 - l1, l3


def first_sweep(n):
    """log2 of the first (column) sweep length L1 of the R2C of n real samples: the fused split's column 0 holds the
    bins that are multiples of L1. None for the single-kernel sizes (log2 M <= 12)"""
    q = (n // 2).bit_length() - 1
    if 27 <= q <= 30:
        return _plan4(q)[0]
    if 13 <= q <= 20:
        return (q + 1) // 2
    if 21 <= q <= 26:
        return _plan3(q)[0]
    return None


def _raw_first_sweep(n, bits, fmt, window):
    """bits of the raw first sweep when the unpack can be fused (srtb_b200.cu raw_sources_for, lines 1904-1940): 0 for
    8-bit samples, 2 / 4 for packed ones, None when the unpack kernel runs first"""
    if window != 0 or n < (1 << 14):
        return None
    if bits in (2, 4) and fmt == SIMPLE:
        return bits
    if bits in (8, -8) and (fmt in (SIMPLE, INTERLEAVED_2, GZNUPSR_A1_2) or (fmt == NAOCPSR_SNAP1 and bits == -8)):
        return 0
    return None


def _raw_accepts(logl, raw_bits):
    """dispatch_col_raw (srtb_b200.cu lines 837-853): first-sweep lengths with a raw variant"""
    return logl in ((7, 8) if raw_bits else (7, 8, 9, 11))


def tail_routes(L):
    """(s1_route, sk_route) of stream_tail (srtb_b200.cu lines 2116-2154) for rows of L: s1 + chirp on load where a
    waterfall kernel reads the spectrum (chirp_fusable line 1625, long_fusable line 1727), else dedisperse_kernel<true>
    ("unfused"); SK in the eight-point row kernel's epilogue for L = 512, in sk_kernel elsewhere"""
    if L in ROW16:
        return "row16", "row16"
    if L in BIGROW:
        return "bigrow", "bigrow"
    if L in LONG:
        return "long", "long"
    return "unfused", ("row8_512" if L == 512 else "unfused")


def rfi_route(n, C, bits, fmt, path, window=0):
    """((mean_route, "raw" | "unpacked"), s1_route, sk_route) for a block of n samples per stream and C channels.
    path = "block" (process_block and the ring) or "sweep" (the DM sweep, which never takes the sweep-order R2C).
    Restates fft_r2c_with_power_mean (srtb_b200.cu lines 1251-1331), r2c_stream (lines 2093-2106) and
    r2c_sweep_order (lines 2068-2076); TMA descriptors are taken to be available and the library's buffers 16-byte
    aligned, as they are on an H100."""
    assert path in ("block", "sweep")
    nc = n // 2
    L = nc // min(C, nc)
    q = nc.bit_length() - 1
    raw = _raw_first_sweep(n, bits, fmt, window)
    if path == "block" and raw == 0 and L == (1 << 14) and nc == (1 << 25):
        mean = ("rows_split", "raw")
    elif 27 <= q <= 30:
        mean = ("fixup4", "raw" if raw is not None and _raw_accepts(_plan4(q)[0], raw) else "unpacked")
    else:
        if 13 <= q <= 20:
            l1, last = (q + 1) // 2, q - (q + 1) // 2
        elif 21 <= q <= 26:
            l1, _, last = _plan3(q)
        else:
            l1, last = None, None
        if last is not None and 6 <= last <= 8:
            name = "fixup2" if q <= 20 else "fixup3"
            mean = (name, "raw" if raw is not None and _raw_accepts(l1, raw) else "unpacked")
        else:
            mean = ("post", "unpacked")     # the raw route needs the fused split: the unpack kernel runs first
    return (mean,) + tail_routes(L)


# ------------------------------------------------------------------------------------------------------- the truth
def _abs2(x):
    return x.real * x.real + x.imag * x.imag


def s1_truth(X, avg_thr, bins=()):
    """(mask, limit, pw) of the s1 stage in float64 for the spectrum X = bins 0 .. Nc - 1 of the R2C: the mean of
    |X|^2 over all Nc bins is taken before the manual ranges are zeroed (the reference's order), the limit is
    float64(float32(avg_thr)) * mean, and mask = pw > limit OR-ed with the manual bins (lo, hi), inclusive."""
    pw = _abs2(X)
    limit = float(np.float32(avg_thr)) * float(pw.mean())
    mask = pw > limit
    for lo, hi in bins:
        mask[lo:hi + 1] = True
    return mask, limit, pw


def sk_truth(spec):
    """L * sum p^2 / (sum p)^2 of every row of spec [C][L] over all L time samples (not the detector's ts_count); an
    all-zero row gives NaN, which no window test rejects"""
    p = _abs2(spec)
    with np.errstate(invalid="ignore", divide="ignore"):
        return spec.shape[-1] * (p * p).sum(-1) / p.sum(-1) ** 2


def sk_window(thr, M):
    """(lo, hi) of sk_bounds (srtb_b200.cu lines 1502-1507) in float32 arithmetic: thr and 2 - thr ordered, each
    scaled by (M - 1) / (M + 1) and shifted by 1 (spectrum/rfi_mitigation.hpp of the reference, lines 300-306)"""
    M_ = np.float32(M)
    hi, lo = np.float32(thr), np.float32(2) - np.float32(thr)
    if lo > hi:
        lo, hi = hi, lo
    f = (M_ - np.float32(1)) / (M_ + np.float32(1))
    return float(lo * f + np.float32(1)), float(hi * f + np.float32(1))


def _fft_rows(y):
    if isinstance(y, np.ndarray):
        return np.fft.fft(y.astype(np.complex128), axis=-1)
    import torch
    return torch.fft.fft(y.to(torch.complex128), dim=-1)


def recover_s1_mask(gspec_rows, X_rows, coef, mean):
    """(zapped, ambiguous) per bin of kept channel rows, from the dynamic spectrum alone. The forward FFT of a channel
    row gives back coef * L * X * chirp for every bin s1 kept and 0 for every bin it zapped, so a bin is zapped iff
    |Y| < 0.5 coef L |X|. Bins with |X|^2 < 1e-6 mean cannot be told apart and are reported as ambiguous.
    gspec_rows [R][L] (complex64), X_rows [R][L] (float64 truth of the same bins)."""
    L = gspec_rows.shape[-1]
    Y = _fft_rows(gspec_rows)
    zapped = _abs2(Y) < 0.25 * (coef * L) ** 2 * _abs2(X_rows)
    ambiguous = _abs2(X_rows) < 1e-6 * mean
    return zapped, ambiguous


@dataclass
class Decisions:
    total: int            # decisions compared
    flips: int            # decided otherwise than the float64 truth
    worst: float          # largest relative distance from the edge among the flips (0 without flips)
    informative: int      # decisions in the band (margin, 100 margin] of their edge


def decision_distance(stat, edges):
    """relative distance of each statistic from its nearest edge: edges = limit (zap above) or (lo, hi) (keep
    inside). NaN statistics are infinitely far."""
    if np.ndim(edges) == 0:
        d = abs(stat / edges - 1)
    else:
        lo, hi = edges
        a, b = abs(stat / lo - 1), abs(stat / hi - 1)
        d = a * (a < b) + b * (a >= b)
    return d.nan_to_num(float("inf")) if hasattr(d, "nan_to_num") else np.nan_to_num(d, nan=np.inf)


def truth_decisions(stat, edges):
    """True = zap: stat > limit, or stat outside [lo, hi]; NaN is kept"""
    if np.ndim(edges) == 0:
        return stat > edges
    lo, hi = edges
    return (stat > hi) | (stat < lo)


def compare_decisions(got, stat, edges, margin, truth=None):
    """got (bool, True = zapped) against the float64 decisions from stat and edges (or `truth` when given, e.g. s1 OR
    the manual ranges, whose statistic is +inf); see Decisions"""
    if truth is None:
        truth = truth_decisions(stat, edges)
    d = decision_distance(stat, edges)
    flip = got != truth
    n_flip = int(flip.sum())
    worst = float(d[flip].max()) if n_flip else 0.0
    informative = int(((d > margin) & (d <= 100 * margin)).sum())
    return Decisions(int(np.prod(tuple(got.shape))), n_flip, worst, informative)


# ------------------------------------------------------------------------------------- inputs with special bins
SPIKES = ("dc", "half", "col0", "generic", "nyquist")
SIGMA = 20.0


def spike_bin(n, kind):
    """the bin a spike of `kind` puts its power into: DC, M / 2, 3 L1 (column 0 of the fused split; 3 * 2^6 when the
    R2C has no split), 3 L1 / 2 (not in column 0) and the Nyquist bin M"""
    M = n // 2
    l1 = first_sweep(n) or 6
    return {"dc": 0, "half": M // 2, "col0": 3 << l1, "generic": 3 << (l1 - 1), "nyquist": M}[kind]


def spike_pattern(n, kind):
    """int16 samples that put about 2 % of an 8-bit block's power (sigma 20) into spike_bin(n, kind): an offset of 2
    (DC), 4 (1, 0, -1, 0, ...) (M / 2), the rounding of 4 cos(2 pi k t / n) (col0, generic; one period tiled) and
    2 (-1)^t (Nyquist)"""
    k = spike_bin(n, kind)
    if kind == "dc":
        return np.full(n, 2, np.int16)
    if kind == "half":
        return np.resize(np.array([4, 0, -4, 0], np.int16), n)
    if kind == "nyquist":
        return np.resize(np.array([2, -2], np.int16), n)
    g = int(np.gcd(n, k))
    period, j = n // g, k // g          # k / n = j / period
    t = np.arange(period)
    return np.resize(np.round(4 * np.cos(2 * np.pi * (j * t % period) / period)).astype(np.int16), n)


def noise_int8(n, seed, sigma=SIGMA):
    rng = np.random.default_rng(seed)
    return np.clip(np.round(rng.standard_normal(n, np.float32) * sigma), -127, 127).astype(np.int8)


def with_spike(noise, kind):
    return np.clip(noise.astype(np.int16) + spike_pattern(noise.size, kind), -128, 127).astype(np.int8)


def spike_fraction(samples, kind):
    """|X_k|^2 of the spike's bin over sum_{k < M} |X_k|^2 of the block's R2C, in float64"""
    X = np.fft.rfft(samples.astype(np.float64))
    pw = _abs2(X)
    return float(pw[spike_bin(samples.size, kind)] / pw[:samples.size // 2].sum())
