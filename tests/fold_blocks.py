"""The fold's float64 restatements at the executable's shapes (C up to 2048 channels, rows of 2^16 samples and more),
computed channel block by channel block with np.bincount so that the host needs a few hundred megabytes, not tens of
gigabytes; the launch geometry srtb_b200_fold and srtb_b200_fold_coherence choose (include/srtb_b200.h); and spectra
with small integer components, on which every term and every sum of either fold is exact in float64.

Same definitions as tests/fold_oracle.py and tests/fold_coherence_oracle.py (the same bins from fold_oracle.bins, the
same kept rule): on integer spectra the results here equal theirs bit for bit, whatever the summation order."""
import numpy as np

import fold_oracle

FOLD_TILE = 2048      # csrc/fold.cuh: time samples per tile
FOLD_MAX_GROUP = 64   # channels per CTA, at most
FOLD_MAX_BINS = 4096


def geometry(rows: int, chan_count: int, fold_count: int, nsub: int, sm_count: int, per_sm: int):
    """(G, K, R, ntiles, finish) of a fold call as include/srtb_b200.h states them: G the largest divisor of
    chan_count / nsub up to 64, K = rows chan_count / G CTAs (rows: the streams of srtb_b200_fold, 1 for
    srtb_b200_fold_coherence), ntiles = ceil(fold_count / 2048), R = min(ntiles, max(1, floor(per_sm SMs / K))) tile
    ranges (per_sm: 4 for the fold, 2 for the coherence fold), and whether fold_finish_kernel runs: (chan_count / nsub
    / G) R > 1"""
    csub = chan_count // nsub
    G = max(d for d in range(1, min(csub, FOLD_MAX_GROUP) + 1) if csub % d == 0)
    K = rows * chan_count // G
    ntiles = -(-fold_count // FOLD_TILE)
    R = min(ntiles, max(1, (per_sm * sm_count) // K))
    return G, K, R, ntiles, (csub // G) * R > 1


def integer_spectra(streams: int, C: int, L: int, seed: int):
    """[C][L] complex64 spectra whose components are integers in [-64, 63]: every |x|^2 and every product of two
    components is exact in fp32 and float64, and every float64 sum stays far below 2^53. Stream s has whole rows zeroed
    at channels 3 + s and C - 1 - 2s (a different pair in each stream), and channel 5 + s zero at sample 0 only: the
    kept rule looks at sample 0 alone, so that channel is not kept although its other samples are folded. No other
    channel is zero at sample 0"""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(streams):
        x = np.empty((C, L), np.complex64)
        v = x.view(np.float32).reshape(C, L, 2)
        for c0 in range(0, C, 256):  # random bytes in slices: a 2^28-sample stream needs no large temporary
            part = v[c0:c0 + 256]
            part[...] = (np.frombuffer(rng.bytes(part.size), np.int8) >> 1).reshape(part.shape)
        first = x[:, 0]
        first[first == 0] = 1  # every channel kept but the masked ones
        for c in (3 + s, C - 1 - 2 * s):
            x[c] = 0
        x[5 + s, 0] = 0
        out.append(x)
    return out


def _channel_power(x, c0, c1, F):
    z = x[c0:c1, :F]
    return z.real.astype(np.float64) ** 2 + z.imag.astype(np.float64) ** 2


def _fine(F: int, phase, nbins):
    """the bins of j < F at the finest nbin requested, and the factor each coarser nbin groups: for powers of two,
    floor(f nbin) = floor(f 4096) >> log2(4096 / nbin) exactly (f nbin is an exact scaling of f 4096), which is checked
    against fold_oracle.bins for every nbin"""
    top = max(nbins)
    bn = fold_oracle.bins(*phase, top, F)
    for nb in nbins:
        assert top % nb == 0 and (top // nb) & (top // nb - 1) == 0, (top, nb)
        assert np.array_equal(fold_oracle.bins(*phase, nb, F), bn // (top // nb)), nb
    return top, bn


def _by_channel(weights_of, n_out, C, F, top, bn, block):
    """n_out arrays [C][top] float64: each channel's sum per bin of the i-th array weights_of(c0, c1) returns
    ([c1 - c0][F] each)"""
    out = [np.zeros((C, top), np.float64) for _ in range(n_out)]
    for c0 in range(0, C, block):
        c1 = min(C, c0 + block)
        idx = (np.arange(c1 - c0)[:, None] * top + bn[None, :]).ravel()
        for o, w in zip(out, weights_of(c0, c1)):
            o[c0:c1] = np.bincount(idx, weights=w.ravel(), minlength=(c1 - c0) * top).reshape(-1, top)
    return out


def _reduce(per_channel, top, nbin, nsub):
    C = per_channel.shape[0]
    return per_channel.reshape(C, nbin, top // nbin).sum(axis=2).reshape(nsub, C // nsub, nbin).sum(axis=1)


def _nonzero_first(x):
    f = x[:, 0]
    return (f.real.astype(np.float32) ** 2 + f.imag.astype(np.float32) ** 2) != 0


def fold_many(spectra, F: int, phase, cases, block: int = 64):
    """fold_oracle.fold(spectra, F, phase, nbin, nsub) for every (nsub, nbin) in cases, each channel's samples read
    once: {(nsub, nbin): (profile [S][nsub][nbin], hits [nbin] uint64, kept [S][nsub] uint32)}"""
    top, bn = _fine(F, phase, [nb for _, nb in cases])
    C = spectra[0].shape[0]
    per = [_by_channel(lambda c0, c1, x=x: [_channel_power(x, c0, c1, F)], 1, C, F, top, bn, block)[0]
           for x in spectra]
    first = [_nonzero_first(x) for x in spectra]
    out = {}
    for nsub, nbin in cases:
        hits = np.bincount(bn // (top // nbin), minlength=nbin).astype(np.uint64)
        prof = np.stack([_reduce(p, top, nbin, nsub) for p in per])
        kept = np.stack([nz.reshape(nsub, C // nsub).sum(axis=1) for nz in first]).astype(np.uint32)
        out[(nsub, nbin)] = prof, hits, kept
    return out


def fold_coherence_many(x, y, F: int, phase, cases, block: int = 64):
    """fold_coherence_oracle.fold_coherence(x, y, F, phase, nbin, nsub) for every (nsub, nbin) in cases:
    {(nsub, nbin): (coherence [4][nsub][nbin], abs_terms [4][nsub][nbin], hits [nbin] uint64, kept [nsub] uint32)}"""
    top, bn = _fine(F, phase, [nb for _, nb in cases])
    C = x.shape[0]
    keep = _nonzero_first(x) & _nonzero_first(y)

    def parts(c0, c1):  # AA, BB, CR, CI, then the sums of the absolute values of their terms
        k = keep[c0:c1, None]
        xs, ys = x[c0:c1, :F], y[c0:c1, :F]
        xr, xi = xs.real.astype(np.float64) * k, xs.imag.astype(np.float64) * k
        yr, yi = ys.real.astype(np.float64) * k, ys.imag.astype(np.float64) * k
        terms = [(xr * xr, xi * xi), (yr * yr, yi * yi), (xr * yr, xi * yi), (xi * yr, -(xr * yi))]
        return [u + v for u, v in terms] + [np.abs(u) + np.abs(v) for u, v in terms]

    per = _by_channel(parts, 8, C, F, top, bn, block)
    coh, mag = per[:4], per[4:]
    out = {}
    for nsub, nbin in cases:
        hits = np.bincount(bn // (top // nbin), minlength=nbin).astype(np.uint64)
        out[(nsub, nbin)] = (np.stack([_reduce(c, top, nbin, nsub) for c in coh]),
                             np.stack([_reduce(m, top, nbin, nsub) for m in mag]), hits,
                             keep.reshape(nsub, C // nsub).sum(axis=1).astype(np.uint32))
    return out


def fold_error_bound(want, terms):
    """the largest |got - want| of a correct srtb_b200_fold against a float64 oracle of the same spectrum (module
    docstring of tests/test_gpu_fold_exact.py): (2u + u^2 + (2 n + 1) 2^-53) (1 + 2^-20) want, u = 2^-24, with n the
    terms each output adds (the subband's channels times hits of the bin)"""
    u = 2.0 ** -24
    return (2 * u + u * u + (2.0 * terms + 1) * 2.0 ** -53) * (1 + 2.0 ** -20) * want


def noise_recording(path, streams: int, N: int, R: int, C: int, last_valid: int, seed: int, rfi_block: int,
                    rfi_channels) -> int:
    """an 8-bit recording of noise (sigma 20 per stream) in blocks of N samples per stream that step by N - R: four
    full blocks and a fifth of last_valid samples. One stream is written as `simple`; two in the naocpsr_snap1 layout
    (two samples of stream 0, then two of stream 1), so last_valid must be even. Block rfi_block alone carries, inside
    its own share (past the R samples the block before it also reads, before the next block's start), a burst of
    band-limited noise N / 20 samples long in the channels rfi_channels = (lo, hi) of C, 20 times the noise's power
    there: about 11 times the kurtosis of noise, which spectral kurtosis zaps, while the fine bins' mean power only
    doubles. Returns the samples per stream"""
    step = N - R
    n = 4 * step + last_valid
    lo, hi = rfi_channels
    rng = np.random.default_rng(seed)
    q = []
    for _ in range(streams):
        v = rng.standard_normal(n) * 20.0
        nb = N // 20
        at = rfi_block * step + R + N // 4
        assert at + nb <= (rfi_block + 1) * step
        spec = np.fft.rfft(rng.standard_normal(nb))
        chan = np.arange(spec.size) * (2 * C) / nb  # baseband frequency in channels
        spec[(chan < lo) | (chan >= hi)] = 0
        burst = np.fft.irfft(spec, n=nb)
        v[at:at + nb] += burst * (np.sqrt(20 * 400.0 * (hi - lo) / C) / burst.std())
        q.append(np.clip(np.rint(v), -127, 127).astype(np.int8))
    if streams == 1:
        q[0].tofile(path)
    else:
        assert streams == 2 and n % 2 == 0
        raw = np.empty(2 * n, np.int8)
        raw.reshape(-1, 4)[:, 0:2] = q[0].reshape(-1, 2)
        raw.reshape(-1, 4)[:, 2:4] = q[1].reshape(-1, 2)
        raw.tofile(path)
    return n
