"""float64 restatement of srtb_b200_fold_coherence (include/srtb_b200.h): the coherence products AA, BB, CR, CI of a
stream pair, folded with the bins of tests/fold_oracle.py over the channels kept in both streams."""
import numpy as np

import fold_oracle


def kept_mask(x, y):
    """channels kept in both streams: |X[c][0]|^2 != 0 and |Y[c][0]|^2 != 0, formed in fp32 as the detector does"""
    def nz(z):
        f = z[:, 0]
        return (f.real.astype(np.float32) ** 2 + f.imag.astype(np.float32) ** 2) != 0
    return nz(x) & nz(y)


def fold_coherence(x, y, fold_count: int, phase_coeffs, nbin: int, nsub: int):
    """x, y: [C][L] complex64. Returns (coherence [4][nsub][nbin] float64 (AA, BB, CR, CI), abs_terms [4][nsub][nbin]
    float64 (the sum of the absolute values of the terms each output adds, the scale of its rounding), hits [nbin]
    uint64, kept [nsub] uint32)"""
    phi0, a, b = phase_coeffs
    bn = fold_oracle.bins(phi0, a, b, nbin, fold_count)
    hits = np.bincount(bn, minlength=nbin).astype(np.uint64)
    C = x.shape[0]
    keep = kept_mask(x, y)
    xs = x[:, :fold_count].astype(np.complex128) * keep[:, None]
    ys = y[:, :fold_count].astype(np.complex128) * keep[:, None]
    xr, xi, yr, yi = xs.real, xs.imag, ys.real, ys.imag
    terms = [(xr * xr, xi * xi), (yr * yr, yi * yi), (xr * yr, xi * yi), (xi * yr, -(xr * yi))]
    coh = np.zeros((4, nsub, nbin), np.float64)
    mag = np.zeros((4, nsub, nbin), np.float64)
    for p, (u, v) in enumerate(terms):
        s = (u + v).reshape(nsub, C // nsub, fold_count).sum(axis=1)
        m = (np.abs(u) + np.abs(v)).reshape(nsub, C // nsub, fold_count).sum(axis=1)
        for k in range(nsub):
            coh[p, k] = np.bincount(bn, weights=s[k], minlength=nbin)
            mag[p, k] = np.bincount(bn, weights=m[k], minlength=nbin)
    kept = keep.reshape(nsub, C // nsub).sum(axis=1).astype(np.uint32)
    return coh, mag, hits, kept
