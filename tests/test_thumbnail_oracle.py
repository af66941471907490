"""The waterfall thumbnail oracle (tests/thumbnail_oracle.py) against the reference's own resample_spectrum_3,
simplify_spectrum_normalize_with_average_value and generate_pixmap, run through the host SYCL shim
(tests/golden/srtb_thumbnail_ref_vectors.npz, written by tests/golden/make_thumbnail_golden.py). The oracle restates
the reference's work-item split for the shim's device limits, so every output is compared bit for bit. No GPU."""
from pathlib import Path

import numpy as np
import pytest

import thumbnail_oracle as T

GOLDEN = Path(__file__).resolve().parent / "golden" / "srtb_thumbnail_ref_vectors.npz"


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", sorted(T.CASES))
def test_oracle_matches_reference_bit_for_bit(golden, name):
    spec = T.case_spectrum(name)
    assert np.sum(T.norm(spec), dtype=np.float64) == golden[f"{name}__input_sum"][0], "seeded input changed"
    raw, avg, inten, pix = T.simplify_spectrum(spec, *T.CASES[name][3:1:-1])
    assert np.array_equal(raw.view(np.uint32), golden[f"{name}__raw"].view(np.uint32))
    assert avg.view(np.uint32) == golden[f"{name}__average"].view(np.uint32)[0]
    assert np.array_equal(inten.view(np.uint32), golden[f"{name}__intensity"].view(np.uint32))
    assert np.array_equal(pix, golden[f"{name}__pixmap"])


def test_impulse_exposes_the_weights(golden):
    """one non-zero cell (|x|^2 = 25) at (r, c): pixel (y2, x2) reads 25 * wy(y2, r) * wx(x2, c), where w is the cell's
    weight in that pixel's extent: 1 inside [lo, hi), wl on lo - 1, wh on hi, both edge weights when lo - 1 == hi"""
    C, L, H, W, _ = T.CASES["impulse"]
    spec = T.case_spectrum("impulse")
    (r, c), = np.argwhere(spec != 0)

    def weights(n_out, n_in, cell):
        lo, hi, wl, wh = T.extents(n_out, n_in)
        w = np.zeros(n_out, np.float32)
        w += np.where((wl > 0) & (lo - 1 == cell), wl, 0)
        w += np.where((lo <= cell) & (cell < hi), 1, 0).astype(np.float32)
        w += np.where((wh > 0) & (hi == cell), wh, 0)
        return w

    wy, wx = weights(H, C, r), weights(W, L, c)
    expect = (np.float32(25) * wx[None, :]) * wy[:, None]  # x sum first, then the y weight, as the reference does
    assert np.array_equal(golden["impulse__raw"].view(np.uint32), expect.astype(np.float32).view(np.uint32))
    assert np.count_nonzero(expect) >= 1


def test_extents_cover_every_cell_once():
    """the integer ranges tile the input: summed weights per input cell are 1 when downsampling (exact ratios), and
    every cell is touched; q12: when upsampling, a pixel inside one cell has weight (r - l) + 1"""
    for n_out, n_in in [(128, 1024), (70, 1000), (1920, 16384), (1080, 2048), (120, 50), (64, 24)]:
        lo, hi, wl, wh = T.extents(n_out, n_in)
        tot = np.zeros(n_in, np.float64)
        for i in range(n_out):
            if wl[i] > 0:
                tot[lo[i] - 1] += wl[i]
            tot[lo[i]:hi[i]] += 1
            if wh[i] > 0:
                tot[hi[i]] += wh[i]
        assert np.all(tot > 0)
        if n_in % n_out == 0:
            assert np.all(tot == 1) and np.all(wl == 0) and np.all(wh == 0)
    lo, hi, wl, wh = T.extents(120, 50)
    inside = lo - 1 == hi  # pixel inside one input cell
    assert inside.any()
    a = (np.arange(120, dtype=np.float32) / np.float32(120)) * np.float32(50)
    b = (np.arange(1, 121, dtype=np.float32) / np.float32(120)) * np.float32(50)
    assert np.array_equal((wl + wh)[inside], ((b - a) + np.float32(1))[inside])


def test_tiny_average_is_left_unscaled(golden):
    assert golden["tiny_average__average"][0] <= np.finfo(np.float32).eps
    assert np.array_equal(golden["tiny_average__raw"], golden["tiny_average__intensity"])
