"""The baseband correlator oracle (tests/correlator_oracle.py) against the reference's own correlator.cpp, run through
the host SYCL shim (tests/golden/srtb_correlator_ref_vectors.npz, written by tests/golden/make_correlator_golden.py).
The oracle restates the program with the same naive FFT and the same float operations, so every output is compared
bit for bit. No GPU."""
from pathlib import Path

import numpy as np
import pytest

import correlator_oracle as K

GOLDEN = Path(__file__).resolve().parent / "golden" / "srtb_correlator_ref_vectors.npz"


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", list(K.CASES))
def test_oracle_matches_reference_bit_for_bit(golden, name):
    in_1, in_2 = K.case_inputs(name)
    assert [K.checksum(in_1), K.checksum(in_2)] == golden[f"{name}__input_crc"].tolist(), "seeded input changed"
    got = K.correlate(in_1, in_2)
    ref = golden[f"{name}__out"]
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("name", list(K.CASES))
def test_reference_within_fft_policy_of_float64(golden, name):
    """the reference itself against |ifft(norm A conj(B)) M| in float64: rel-L2 <= 1e-5, max-abs <= 1e-4 RMS"""
    in_1, in_2 = K.case_inputs(name)
    truth = K.truth_float64(in_1, in_2)
    ref = golden[f"{name}__out"].astype(np.float64)
    rms = np.sqrt(np.mean(truth ** 2))
    assert np.linalg.norm(ref - truth) <= 1e-5 * np.linalg.norm(truth)
    assert np.max(np.abs(ref - truth)) <= 1e-4 * rms


def test_odd_input_size_scales_by_the_odd_size(golden):
    """q13: a 2^k + 1-byte pair is read as 2^k samples but scaled by (2^k + 1)^-1.5, as the reference does"""
    in_1, in_2 = K.case_inputs("odd_1025")
    even = K.correlate(in_1[:1024], in_2[:1024])
    odd = golden["odd_1025__out"]
    assert K.norm_coeff(1025) != K.norm_coeff(1024)
    ratio = odd.astype(np.float64) / even.astype(np.float64)
    assert np.allclose(ratio, (1024 / 1025) ** 1.5, rtol=1e-6)


def test_unequal_sizes_use_the_smaller_file(golden):
    in_1, in_2 = K.case_inputs("unequal_9000_4097")
    assert np.array_equal(golden["unequal_9000_4097__out"].view(np.uint32),
                          K.correlate(in_1[:4097], in_2).view(np.uint32))


def test_constant_input_is_dc_only(golden):
    """two constant inputs have only a DC bin: every lag of the output has the same magnitude"""
    out = golden["const__out"]
    m, n = K.sizes(4096)
    expect = float(K.norm_coeff(4096)) * (200.0 * n) * (57.0 * n)
    assert np.allclose(out, expect, rtol=1e-6)


def test_known_delay_peaks_where_float64_puts_it(golden):
    """input 2 is input 1 rolled by DELAY samples: the M-point inverse of the first M bins peaks at lag -DELAY / 2
    (mod M)"""
    in_1, in_2 = K.case_inputs("delay")
    m, _ = K.sizes(in_1.size)
    out = golden["delay__out"]
    assert int(np.argmax(out)) == int(np.argmax(K.truth_float64(in_1, in_2))) == (-K.DELAY // 2) % m
