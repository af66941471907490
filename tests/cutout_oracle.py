"""Float64 restatement of the candidate cut-outs (srtb_b200_candidate_cutouts, include/srtb_b200.h), for the tests.

For S spectra x_s [C][L], coherently dedispersed at `dm`, with data in j < ts = L - time_reserved_count:

    P(c, j)   = sum_s |x_s[c][j]|^2 for 0 <= j < ts when channel c is kept (|x_s[c][0]|^2 != 0 in float32 in every
                stream), else 0
    k[c]      = (1/f(c)^2 - 1/f_ref^2) sample_rate / (2C) 4.148808e3        (the incoherent search's, in float64)
    s(d, c)   = round_half_away(((float64(d) - float64(dm)) k[c]) / q)
    t0        = center - (W/2) q,  D(c, m) = sum_{u<q} P(c, t0 + m q + u)
    ft[k][i]  = sum over the C/nsub channels of subband k of D(c, i + s(dm_req, c))
    DM_r      = float32(dm_req + halfwidth (r - n_rows/2) / (n_rows/2)), dm_req for n_rows == 1
    dmt[r][i] = sum_c D(c, i + s(DM_r, c))

The sums here are float64; the library adds in float32 in the order above. Every term is non-negative, so a float32
result lies within (adds + 2) 2^-24 of the float64 sum relatively (`bound`).
"""
from __future__ import annotations

import numpy as np

from incoherent_oracle import DISPERSION_CONSTANT, round_half_away


def k_table(chan_count: int, freq_low: float, bandwidth: float, sample_rate: float) -> np.ndarray:
    """k [C] in float64, in the library's order of operations"""
    fl, bw, sr = (float(np.float32(v)) for v in (freq_low, bandwidth, sample_rate))
    f_ref = float(np.float32(np.float32(freq_low) + np.float32(bandwidth)))
    scale = sr / (2.0 * chan_count)
    c = np.arange(chan_count, dtype=np.float64)
    f = fl + bw * (c + 0.5) / chan_count
    return (1.0 / (f * f) - 1.0 / (f_ref * f_ref)) * scale * DISPERSION_CONSTANT


def row_dms(dm_req: float, halfwidth: float, n_rows: int) -> np.ndarray:
    """DM_r [n_rows] float32"""
    if n_rows == 1:
        return np.array([dm_req], np.float32)
    h = n_rows // 2
    r = np.arange(n_rows, dtype=np.float64)
    return (float(np.float32(dm_req)) + float(np.float32(halfwidth)) * (r - h) / h).astype(np.float32)


def shifts(k: np.ndarray, dm: float, dms, q: int) -> np.ndarray:
    """s [len(dms)][C] int64"""
    d = np.asarray([float(np.float32(v)) for v in np.atleast_1d(dms)], np.float64) - float(np.float32(dm))
    return round_half_away((d[:, None] * k[None, :]) / float(q))


def kept_channels(spectra) -> np.ndarray:
    """[C] bool: |x_s[c][0]|^2 != 0 in float32 in every stream"""
    keep = None
    for x in spectra:
        x0 = np.asarray(x[:, 0], np.complex64)
        p = x0.real * x0.real + x0.imag * x0.imag  # float32, no contraction
        keep = (p != 0) if keep is None else keep & (p != 0)
    return keep


def power(spectra, time_reserved_count: int) -> np.ndarray:
    """P [C][ts] in float64 (masked channels 0)"""
    ts = spectra[0].shape[1] - time_reserved_count
    p = np.zeros((spectra[0].shape[0], ts), np.float64)
    for x in spectra:
        xs = np.asarray(x[:, :ts]).astype(np.complex128)
        p += xs.real * xs.real + xs.imag * xs.imag
    p[~kept_channels(spectra)] = 0
    return p


def decimated(P: np.ndarray, t0: int, q: int, m_lo: int, m_hi: int) -> np.ndarray:
    """D [C][m_hi - m_lo]: D(c, m) for m_lo <= m < m_hi, zero outside [0, ts)"""
    C, ts = P.shape
    a, b = t0 + m_lo * q, t0 + m_hi * q
    buf = np.zeros((C, b - a), np.float64)
    lo, hi = max(a, 0), min(b, ts)
    if hi > lo:
        buf[:, lo - a:hi - a] = P[:, lo:hi]
    return buf.reshape(C, m_hi - m_lo, q).sum(axis=2)


def cutout(P: np.ndarray, k: np.ndarray, dm: float, center: int, dm_req: float, halfwidth: float, q: int, W: int,
           nsub: int, n_rows: int):
    """(ft [nsub][W], dmt [n_rows][W], row DMs [n_rows] float32) of one request, float64"""
    C = P.shape[0]
    dms = row_dms(dm_req, halfwidth, n_rows)
    s_rows = shifts(k, dm, dms, q)
    s_req = shifts(k, dm, [dm_req], q)[0]
    lo = int(min(s_rows.min(), s_req.min()))
    hi = int(max(s_rows.max(), s_req.max()))
    t0 = center - (W // 2) * q
    D = decimated(P, t0, q, lo, hi + W)
    i = np.arange(W)
    cc = np.arange(C)[:, None]
    img = D[cc, i[None, :] + (s_req - lo)[:, None]]
    ft = img.reshape(nsub, C // nsub, W).sum(axis=1)
    dmt = np.empty((n_rows, W), np.float64)
    for r in range(n_rows):
        dmt[r] = D[cc, i[None, :] + (s_rows[r] - lo)[:, None]].sum(axis=0)
    return ft, dmt, dms


def cutouts(spectra, time_reserved_count: int, freq_low: float, bandwidth: float, sample_rate: float, dm: float,
            requests, W: int, nsub: int, n_rows: int):
    """every request (center, dm_req, halfwidth, q): (ft [n][nsub][W], dmt [n][n_rows][W], row DMs [n][n_rows])"""
    P = power(spectra, time_reserved_count)
    k = k_table(P.shape[0], freq_low, bandwidth, sample_rate)
    out = [cutout(P, k, dm, int(c), d, h, int(q), W, nsub, n_rows) for c, d, h, q in requests]
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]), np.stack([o[2] for o in out]))


def bound(streams: int, channels: int, q: int) -> float:
    """relative bound of a float32 sum of `channels` channels of q samples of `streams` streams' powers"""
    return (streams + q + channels + 2) * 2.0 ** -24 * 1.01
