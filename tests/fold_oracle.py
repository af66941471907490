"""float64 restatement of the fold (include/srtb_b200.h, "folding at a known pulsar period"): the phase model, each
spectrum sample's bin, and one call's profile, hits and kept."""
import numpy as np


def phase(period: float, period_derivative: float, sample_rate: float, samples_per_spectrum_sample: int,
          first_sample: int):
    """(phi0, a, b) with the operations of srtb_b200_fold_phase, in the same order"""
    t0 = float(first_sample) / sample_rate
    q = period_derivative / (period * period)
    phi = t0 / period - (0.5 * q) * (t0 * t0)
    delta = float(samples_per_spectrum_sample) / sample_rate
    return phi - np.floor(phi), (1.0 / period - q * t0) * delta, (-0.5 * q) * (delta * delta)


def bins(phi0: float, a: float, b: float, nbin: int, count: int) -> np.ndarray:
    """bin of every j < count: p = (phi0 + a j) + b (j j), f = p - floor(p), min(floor(f nbin), nbin - 1); numpy's
    element-wise float64 operations round each step, as the device does"""
    j = np.arange(count, dtype=np.float64)
    p = (phi0 + a * j) + b * (j * j)
    f = p - np.floor(p)
    return np.minimum(np.floor(f * float(nbin)), nbin - 1).astype(np.int64)


def fold(spectra, fold_count: int, phase_coeffs, nbin: int, nsub: int):
    """spectra: list of [C][L] complex64 arrays. Returns (profile [S][nsub][nbin] float64, hits [nbin] uint64,
    kept [S][nsub] uint32)"""
    phi0, a, b = phase_coeffs
    bn = bins(phi0, a, b, nbin, fold_count)
    hits = np.bincount(bn, minlength=nbin).astype(np.uint64)
    S = len(spectra)
    C = spectra[0].shape[0]
    profile = np.zeros((S, nsub, nbin), np.float64)
    kept = np.zeros((S, nsub), np.uint32)
    for s, x in enumerate(spectra):
        xs = x[:, :fold_count]
        pw = xs.real.astype(np.float64) ** 2 + xs.imag.astype(np.float64) ** 2
        sub = pw.reshape(nsub, C // nsub, fold_count).sum(axis=1)          # [nsub][F]
        for k in range(nsub):
            profile[s, k] = np.bincount(bn, weights=sub[k], minlength=nbin)
        first = x[:, 0]
        nz = (first.real.astype(np.float32) ** 2 + first.imag.astype(np.float32) ** 2) != 0
        kept[s] = nz.reshape(nsub, C // nsub).sum(axis=1)
    return profile, hits, kept
