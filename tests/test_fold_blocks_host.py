"""tests/fold_blocks.py against the plain restatements it stands in for at large shapes: on integer spectra its channel
-blocked folds equal tests/fold_oracle.py and tests/fold_coherence_oracle.py bit for bit, on random floats to float64
rounding; and its launch geometry at the shapes tests/test_gpu_fold_exact.py relies on."""
import numpy as np
import pytest

import fold_blocks as fb
import fold_coherence_oracle as fco
import fold_oracle as fo

C_, L_, F_ = 64, 5000, 4321
PHASE = fo.phase(0.0015578064924, 1.05e-19, 62.5e6, 2 * C_, (1 << 40) + 4321)
CASES = [(1, 1), (1, 4096), (8, 64), (8, 1024), (C_, 1), (C_, 4096)]


def test_integer_spectra_are_integers_with_their_masks():
    xs = fb.integer_spectra(2, C_, L_, seed=1)
    for s, x in enumerate(xs):
        v = x.view(np.float32)
        assert np.array_equal(v, np.rint(v)) and np.abs(v).max() == 64
        assert not x[3 + s].any() and not x[C_ - 1 - 2 * s].any()
        assert x[5 + s, 0] == 0 and x[5 + s, 1:].any()


@pytest.mark.parametrize("block", [1, 7, 64])
def test_fold_many_equals_fold_oracle_on_integers(block):
    xs = fb.integer_spectra(2, C_, L_, seed=2)
    got = fb.fold_many(xs, F_, PHASE, CASES, block=block)
    for (nsub, nbin), (prof, hits, kept) in got.items():
        wprof, whits, wkept = fo.fold(xs, F_, PHASE, nbin, nsub)
        assert np.array_equal(prof, wprof) and np.array_equal(hits, whits) and np.array_equal(kept, wkept)
        assert kept.dtype == wkept.dtype and hits.dtype == whits.dtype


@pytest.mark.parametrize("block", [1, 64])
def test_fold_coherence_many_equals_oracle_on_integers(block):
    x, y = fb.integer_spectra(2, C_, L_, seed=3)
    y[9] = 0
    got = fb.fold_coherence_many(x, y, F_, PHASE, CASES, block=block)
    for (nsub, nbin), (coh, mag, hits, kept) in got.items():
        wcoh, wmag, whits, wkept = fco.fold_coherence(x, y, F_, PHASE, nbin, nsub)
        assert np.array_equal(coh, wcoh) and np.array_equal(mag, wmag)
        assert np.array_equal(hits, whits) and np.array_equal(kept, wkept)
        assert int(kept.sum()) == C_ - 7  # 3, 4, 5, 6, 9, C - 1 and C - 3 are masked in X or Y


def test_random_floats_agree_to_float64_rounding():
    rng = np.random.default_rng(4)
    x, y = [(rng.standard_normal((C_, L_)) + 1j * rng.standard_normal((C_, L_))).astype(np.complex64)
            for _ in range(2)]
    for (nsub, nbin), (prof, hits, kept) in fb.fold_many([x, y], F_, PHASE, CASES).items():
        wprof, whits, wkept = fo.fold([x, y], F_, PHASE, nbin, nsub)
        assert np.array_equal(hits, whits) and np.array_equal(kept, wkept)
        assert np.all(np.abs(prof - wprof) <= 1e-12 * wprof)
    for (nsub, nbin), (coh, mag, hits, kept) in fb.fold_coherence_many(x, y, F_, PHASE, CASES).items():
        wcoh, wmag, _, _ = fco.fold_coherence(x, y, F_, PHASE, nbin, nsub)
        assert np.all(np.abs(coh - wcoh) <= 1e-13 * wmag)


def test_bins_not_a_power_of_two_are_refused():
    with pytest.raises(AssertionError):
        fb.fold_many([np.ones((4, 100), np.complex64)], 100, PHASE, [(1, 7), (1, 64)])


def test_error_bound_is_the_derived_one():
    u = 2.0 ** -24
    assert fb.fold_error_bound(1.0, 0) == pytest.approx(2 * u + u * u + 2.0 ** -53, rel=1e-5)
    assert fb.fold_error_bound(3.0, 1e6) == pytest.approx(3 * (2 * u + (2e6 + 1) * 2.0 ** -53), rel=1e-5)
    assert fb.fold_error_bound(1.0, 1e6) < 1e-5 / 40


def test_launch_geometry_at_the_h100_sm_count():
    """(G, K, R, ntiles, finish) at 132 SMs for the shapes of tests/test_gpu_fold_exact.py"""
    sm = 132
    assert fb.geometry(1, 2048, 15590, 1, sm, 4) == (64, 32, 8, 8, True)       # one tile per range
    assert fb.geometry(1, 2048, 15590, 2048, sm, 4) == (1, 2048, 1, 8, False)  # 8 tiles per CTA, no finish
    assert fb.geometry(2, 2048, 15590, 64, sm, 4) == (32, 128, 4, 8, True)
    assert fb.geometry(1, 256, 7949, 256, sm, 4) == (1, 256, 2, 4, True)       # two tiles per range, G = 1
    assert fb.geometry(1, 2048, 64742, 1, sm, 4) == (64, 32, 16, 32, True)     # two tiles per range, G = 64
    assert fb.geometry(1, 2048, 64742, 1, sm, 2) == (64, 32, 8, 32, True)
    assert fb.geometry(1, 256, 7949, 256, sm, 2) == (1, 256, 1, 4, False)
    assert fb.geometry(1, 96, 100, 3, sm, 4) == (32, 3, 1, 1, False)            # the largest divisor up to 64
    assert fb.geometry(1, 96 * 3, 100, 3, sm, 4)[0] == 48


@pytest.mark.parametrize("streams", [1, 2])
def test_noise_recording_layout_and_burst(tmp_path, streams):
    """the file holds 4 (N - R) + last samples per stream in the format's layout; the burst raises the power of its
    channels inside block 2's own share only"""
    N, R, C, last = 1 << 15, 1 << 11, 16, 20002
    path = tmp_path / "r.bin"
    n = fb.noise_recording(path, streams, N, R, C, last, seed=7, rfi_block=2, rfi_channels=(5, 7))
    raw = np.fromfile(path, np.int8)
    assert n == 4 * (N - R) + last and raw.size == streams * n
    s0 = raw.reshape(-1, 4)[:, 0:2].ravel() if streams == 2 else raw
    step, nb = N - R, N // 20
    at = 2 * step + R + N // 4

    def band_power(seg, lo, hi):
        p = np.abs(np.fft.rfft(seg.astype(np.float64))) ** 2
        chan = np.arange(p.size) * (2 * C) / seg.size
        return p[(chan >= lo) & (chan < hi)].mean()

    burst, quiet = s0[at:at + nb], s0[at - 2 * nb:at - nb]
    assert band_power(burst, 5, 7) > 10 * band_power(quiet, 5, 7)
    assert band_power(burst, 9, 15) < 1.5 * band_power(quiet, 9, 15)
    assert at - 2 * nb > 2 * step + R and at + nb <= 3 * step
