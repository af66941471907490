"""The float64 detector truth (detector_truth.py) checked on the CPU: its boxcars against direct windowed sums, its exact
header fields against the CPU oracle on every edge geometry the GPU module runs, and the oracle's fp32 values inside
the truth's bounds (widened for the oracle's pairwise fp32 sums and serial fp32 scan)."""
import numpy as np
import pytest

import detector_truth as dt

SNR, CHAN_THR = 6.0, 0.9

# (C, L, reserved, max_boxcar) of the per-pipe detector. ts_count = L - reserved, or L when reserved >= L.
# Aimed at colsum_final_scan_kernel's branches (tiles of 4 x 1024 linked by an fp64 carry, scalar tails, several
# column groups per CTA above 32 x SMs, empty chunk groups, the zero count's grid-stride loop at ts_count <= 32 and
# C > 1024) and at detect_boxcar_kernel's ladder end (ts_count = 2^k + 1 leaves a last series of length 1).
PIPE_CASES = [
    (33, 1, 0, 4),            # ts 1
    (128, 2, 0, 1),           # ts 2, max_boxcar 1
    (129, 10, 7, 3),          # ts 3, reserved not a multiple of 4, max_boxcar 3
    (1000, 4, 0, 100),        # ts 4; 125 partial rows of 8 channels
    (2048, 5, 5, 0),          # reserved >= L keeps L; max_boxcar 0
    (1, 31, 0, 64),           # one channel: 31 of 32 chunk groups empty; max_boxcar >= ts_count
    (3000, 32, 0, 8),         # grid of one CTA: the zero count walks channels 1024 .. 2999 in its loop
    (3000, 40, 7, 16),        # ts 33: two CTAs, still fewer threads than channels
    (33, 4095, 0, 4095),      # one scan tile minus one
    (128, 4096, 0, 100),      # exactly one tile
    (129, 4097, 0, 4096),     # one tile plus one; the last boxcar has one element
    (1, 8193, 0, 8192),       # three tiles, ladder end 2^13 + 1
    (1000, 12300, 9, 3),      # ts 3 * 4096 + 3
    (33, 20000, 0, 1024),     # ts above 32 x SMs: every CTA walks several column groups
    (2048, 1024, 0, 1),
    (16, 6001, 6001, 5000),   # reserved == L
]
# (batch_size, count_per_batch, max_boxcar) of the v1 detector ([time][frequency])
V1_CASES = [(4095, 64, 4096), (4097, 48, 4096), (32, 3000, 16), (31, 1500, 64)]


def pipe_spectrum(C, L, seed):
    """[C][L] complex64 noise, a broadband pulse (8 time samples x 3 in amplitude), channel 1 zeroed, and for more than
    1024 channels two zeroed channels past the first CTA's 1024 threads"""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((C, L)) + 1j * rng.standard_normal((C, L))).astype(np.complex64)
    x[:, L // 3:L // 3 + 8] *= 3
    if C > 2:
        x[1] = 0
    if C > 1024:
        x[[C // 2 + 1000, C - 1]] = 0
    return x


def v1_spectrum(nt, nf, seed):
    """[time][frequency]: noise, a steady tone (SK zaps it), a zeroed channel, one past 1024 when there are more, and a
    broadband burst"""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((nt, nf)) + 1j * rng.standard_normal((nt, nf))).astype(np.complex64)
    x[:, 5] = 3
    x[:, 11] = 0
    if nf > 1024:
        x[:, nf - 7] = 0
    x[nt // 3:nt // 3 + 4, :] *= 1.6
    return x


def _check_exact(res, t):
    assert int(res.zero_count) == t.zero_count
    assert int(res.time_series_count) == t.time_series_count
    assert bool(res.detect_enabled) == t.detect_enabled
    assert int(res.n_boxcars) == t.n_boxcars
    for b in range(t.n_boxcars):
        assert int(res.boxcar_length[b]) == t.boxcar_length[b]
        assert int(res.series_length[b]) == t.series_length[b]


@pytest.mark.parametrize("n,maxbox", [(1, 8), (2, 8), (5, 4), (33, 64), (4097, 4096), (1000, 100)])
def test_boxcars_equal_direct_windowed_sums(n, maxbox):
    rng = np.random.default_rng(n)
    A = rng.exponential(2.0, n) * 16
    t = dt.truth_from_columns(A, 16, 0, SNR, CHAN_THR, maxbox)
    d = A - A.mean()
    assert np.array_equal(t.series[0], d)
    assert t.boxcar_length == dt.boxcar_lengths(n, maxbox)
    for b, S in zip(t.boxcar_length[1:], t.series[1:]):
        direct = np.convolve(d, np.ones(b), "valid")[1:]   # S_b[i] = d[i+1] + .. + d[i+b]
        assert S.size == n - b == direct.size
        scale = np.abs(d).sum()
        assert np.abs(S - direct).max() <= 1e-12 * scale
    for b in range(t.n_boxcars):
        S = t.series[b]
        assert t.variance[b] == pytest.approx(np.mean(S * S), rel=1e-12)
        assert t.count_lo[b] <= t.count_hi[b]
        assert np.all(t.err[b] > 0)


def test_trimming_enable_and_ladder_rules():
    assert dt.ts_count_for(100, 0) == 100 and dt.ts_count_for(100, 7) == 93
    assert dt.ts_count_for(100, 100) == 100 and dt.ts_count_for(100, 101) == 100
    assert dt.boxcar_lengths(1, 64) == [1] and dt.boxcar_lengths(3, 0) == [1] and dt.boxcar_lengths(3, 1) == [1]
    assert dt.boxcar_lengths(5, 3) == [1, 2] and dt.boxcar_lengths(4097, 10 ** 9)[-1] == 4096
    assert len(dt.boxcar_lengths(1 << 40, 1 << 40)) == 32
    # float(0.9) * float(10) rounds to 9 in fp32: 8 zero channels of 10 leave detection on, 9 switch it off
    assert dt.detect_enabled(8, 10, 0.9) and not dt.detect_enabled(9, 10, 0.9)
    assert not dt.detect_enabled(0, 0, 0.9) and not dt.detect_enabled(5, 5, 0.9)


@pytest.mark.parametrize("C_,L,reserved,maxbox", PIPE_CASES)
def test_truth_matches_oracle_per_pipe(oracle, C_, L, reserved, maxbox):
    x = pipe_spectrum(C_, L, seed=C_ * 7919 + L)
    eres, eseries = oracle.signal_detect(x.reshape(-1), L, C_, reserved, SNR, CHAN_THR, maxbox)
    t = dt.signal_detect(x, L, C_, reserved, SNR, CHAN_THR, maxbox)
    _check_exact(eres, t)
    dt.compare(eres, eseries, dt.signal_detect(x, L, C_, reserved, SNR, CHAN_THR, maxbox, fp32_oracle=True))


@pytest.mark.parametrize("nt,nf,maxbox", V1_CASES)
def test_truth_matches_oracle_v1(oracle, nt, nf, maxbox):
    x = v1_spectrum(nt, nf, seed=nt * 31 + nf)
    espec, eres, eseries = oracle.signal_detect_v1(x.reshape(-1), nf, nt, 1.4, SNR, CHAN_THR, maxbox)
    t = dt.signal_detect_v1(espec, nf, nt, SNR, CHAN_THR, maxbox)
    _check_exact(eres, t)
    dt.compare(eres, eseries, dt.signal_detect_v1(espec, nf, nt, SNR, CHAN_THR, maxbox, fp32_oracle=True))


@pytest.mark.parametrize("zero_rows", [8, 9])
def test_truth_matches_oracle_at_the_channel_threshold(oracle, zero_rows):
    C_, L = 10, 64
    x = pipe_spectrum(C_, L, seed=zero_rows)
    x[:zero_rows] = 0
    eres, _ = oracle.signal_detect(x.reshape(-1), L, C_, 0, SNR, CHAN_THR, 16)
    t = dt.signal_detect(x, L, C_, 0, SNR, CHAN_THR, 16)
    _check_exact(eres, t)
    assert t.detect_enabled == (zero_rows == 8)


def test_constant_rows_give_zero_variance(oracle):
    """rows constant in time with small integer powers: every column sum, the mean and d = 0 are exact in fp32"""
    C_, L = 10, 5000
    x = np.repeat((np.arange(C_) % 3 + 1).astype(np.complex64)[:, None], L, axis=1)
    t = dt.signal_detect(x, L, C_, 0, SNR, CHAN_THR, 64)
    eres, eseries = oracle.signal_detect(x.reshape(-1), L, C_, 0, SNR, CHAN_THR, 64)
    _check_exact(eres, t)
    assert t.n_boxcars == 7
    for b in range(t.n_boxcars):
        assert not t.series[b].any() and t.variance[b] == 0 and t.threshold[b] == 0
        assert eres.variance[b] == 0 and eres.threshold[b] == 0 and eres.signal_count[b] == 0


def test_bounds_reject_a_wrong_count_and_a_shifted_series(oracle):
    """the comparison is not vacuous: a count off by the pulse, or a series moved by ten times its bound, fails"""
    C_, L = 64, 4096
    x = pipe_spectrum(C_, L, seed=3)
    eres, eseries = oracle.signal_detect(x.reshape(-1), L, C_, 0, SNR, CHAN_THR, 64)
    t = dt.signal_detect(x, L, C_, 0, SNR, CHAN_THR, 64, fp32_oracle=True)
    assert t.count_lo[0] > 0
    dt.compare(eres, eseries, t)
    eres.signal_count[0] = 0
    with pytest.raises(AssertionError):
        dt.compare(eres, None, t)
    eres.signal_count[0] = t.count_lo[0]
    bad = eseries.copy()
    bad[2, 100] += 10 * t.err[2][100]
    with pytest.raises(AssertionError):
        dt.compare(eres, bad, t)
