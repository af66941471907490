"""CPU oracle of the baseband correlator (the reference's userspace/src/correlator.cpp) — TEST INFRASTRUCTURE ONLY.

The unpack and the naive R2C / backward C2C come from the C++ oracle (oracle_lib); the cross spectrum (1) and the
magnitude (3) are numpy float32, one rounding per operation, in the reference's order. CASES are the seeded input
pairs of tests/golden/srtb_correlator_ref_vectors.npz (written by tests/golden/make_correlator_golden.py)."""
from __future__ import annotations

import zlib

import numpy as np

import oracle_lib

# name: (size_1, size_2, kind, seed); kind: "uniform" bytes, "const" (DC only) or "delay" (input 2 is input 1 rolled
# by DELAY samples)
CASES = {
    "n2": (2, 2, "uniform", 1),
    "n4": (4, 4, "uniform", 2),
    "n8": (8, 8, "uniform", 3),
    "n1k": (1 << 10, 1 << 10, "uniform", 4),
    "n16k": (1 << 14, 1 << 14, "uniform", 5),
    "n32k": (1 << 15, 1 << 15, "uniform", 6),
    "n64k": (1 << 16, 1 << 16, "uniform", 7),
    "odd_9": (9, 9, "uniform", 8),
    "odd_1025": (1025, 1025, "uniform", 9),
    "odd_16385": ((1 << 14) + 1, (1 << 14) + 1, "uniform", 10),
    "unequal_4096_5000": (4096, 5000, "uniform", 11),
    "unequal_9000_4097": (9000, 4097, "uniform", 12),
    "const": (4096, 4096, "const", 13),
    "delay": (1 << 14, 1 << 14, "delay", 14),
}
DELAY = 1000


def case_inputs(name: str) -> tuple[np.ndarray, np.ndarray]:
    """the two seeded unsigned 8-bit inputs of a case, at their full (file) sizes"""
    s1, s2, kind, seed = CASES[name]
    rng = np.random.default_rng(seed)
    if kind == "const":
        return np.full(s1, 200, np.uint8), np.full(s2, 57, np.uint8)
    a = rng.integers(0, 256, max(s1, s2), dtype=np.uint8)
    if kind == "delay":
        b = np.roll(a, DELAY)
        return a[:s1].copy(), b[:s2].copy()
    b = rng.integers(0, 256, s2, dtype=np.uint8)
    return a[:s1].copy(), b


def checksum(x: np.ndarray) -> int:
    return zlib.crc32(np.ascontiguousarray(x).tobytes())


def sizes(input_size: int) -> tuple[int, int]:
    """(complex_count M, real_count) of correlator.cpp:56-57"""
    m = input_size // 2
    return m, 2 * m


def norm_coeff(input_size: int) -> np.float32:
    """float(std::pow(input_size, -1.5)): double pow, one rounding to float (correlator.cpp:59)"""
    return np.float32(float(input_size) ** -1.5)


def cross_spectrum(x1: np.ndarray, x2: np.ndarray, norm: np.float32) -> np.ndarray:
    """(norm X1) conj(X2) as SyclCPLX's float operators compute it: a = norm Re X1, b = norm Im X1, c = Re X2,
    d = -Im X2; (ac - bd, ad + bc), every product and sum rounded to float"""
    x1 = np.ascontiguousarray(x1, np.complex64)
    x2 = np.ascontiguousarray(x2, np.complex64)
    norm = np.float32(norm)
    a, b = x1.real * norm, x1.imag * norm
    c, d = x2.real, -x2.imag
    out = np.empty(x1.shape, np.complex64)
    out.real = a * c - b * d
    out.imag = a * d + b * c
    return out


def magnitude(y: np.ndarray) -> np.ndarray:
    """srtb::abs of a complex float: hypotf(re, im)"""
    return np.hypot(y.real, y.imag).astype(np.float32)


def correlate(in_1: np.ndarray, in_2: np.ndarray) -> np.ndarray:
    """the reference program on two byte arrays of any sizes: M = min(size) // 2 floats"""
    o = oracle_lib.load()
    input_size = min(in_1.size, in_2.size)
    m, n = sizes(input_size)
    x1 = o.fft_r2c(o.unpack(in_1[:n], n, 8))[:m]
    x2 = o.fft_r2c(o.unpack(in_2[:n], n, 8))[:m]
    y = o.fft_c2c(cross_spectrum(x1, x2, norm_coeff(input_size)), -1)
    return magnitude(y)


def truth_float64(in_1: np.ndarray, in_2: np.ndarray) -> np.ndarray:
    """|ifft(norm A conj(B)) M|, A and B the first M bins of the float64 rfft of each input, norm as the program rounds
    it"""
    input_size = min(in_1.size, in_2.size)
    m, n = sizes(input_size)
    a = np.fft.rfft(in_1[:n].astype(np.float64))[:m]
    b = np.fft.rfft(in_2[:n].astype(np.float64))[:m]
    return np.abs(np.fft.ifft(float(norm_coeff(input_size)) * a * np.conj(b)) * m)
