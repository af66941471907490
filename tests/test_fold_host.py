"""CPU checks of folding's host pieces: srtb_b200_fold_phase against the float64 oracle (tests/fold_oracle.py) and
against the phase model itself, the config keys, their start-up rejections, read_file_pipe's block timing and the sink's
accumulator (tests/cpp/test_fold.cpp), and the executable's rejections."""
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import fold_oracle as fo
import srtb_b200

ROOT = Path(__file__).resolve().parent.parent

CASES = [  # period, period derivative, sample rate, 2C, first sample
    (0.7145197, 0.0, 128e6, 4096, 0),
    (0.0893, 1.25e-13, 1e9, 4096, 123456789),
    (0.00575745, -3.4e-15, 62.5e6, 512, (1 << 40) - 4097),
    (1.2, 4e-12, 2e9, 65536, (1 << 40) + 3 * 65536),
    (3e-5, 7e-10, 128e6, 32, 987654321),
]


@pytest.mark.parametrize("case", CASES)
def test_fold_phase_matches_oracle(case):
    got = srtb_b200.fold_phase(*case)
    want = fo.phase(*case)
    assert got == tuple(float(w) for w in want)
    assert 0.0 <= got[0] < 1.0


@pytest.mark.parametrize("case", CASES)
def test_phase_model_follows_the_definition(case):
    """phi0 + a j + b j^2 of a block is the model's phase at t_j, modulo one turn, over several consecutive blocks"""
    P, Pdot, sr, spp, first = case
    P_, Pdot_, sr_ = Fraction(P), Fraction(Pdot), Fraction(sr)
    L = 4096
    for k in range(3):
        fs = first + k * L * spp
        phi0, a, b = srtb_b200.fold_phase(P, Pdot, sr, spp, fs)
        for j in (0, 1, 777, L - 1):
            t = Fraction(fs + spp * j) / sr_
            exact = t / P_ - Pdot_ / (P_ * P_) * t * t / 2
            d = (phi0 + a * j + b * j * j) - float(exact - (exact.numerator // exact.denominator))
            assert abs(d - round(d)) < 1e-9, (k, j, d)


def test_bins_bit_identical_across_blocks():
    """the oracle's bins from the library's coefficients, block after block: every bin in range, the count right, and
    a block's bins continue the previous block's where the blocks meet"""
    P, Pdot, sr, spp = 0.0123456, 3.2e-9, 62.5e6, 128
    F, nbin = 5000, 97
    prev_last = None
    for k in range(4):
        ph = srtb_b200.fold_phase(P, Pdot, sr, spp, k * F * spp)
        assert ph == tuple(float(w) for w in fo.phase(P, Pdot, sr, spp, k * F * spp))
        bn = fo.bins(*ph, nbin, F + 1)
        assert bn.min() >= 0 and bn.max() < nbin
        if prev_last is not None:
            assert bn[0] == prev_last  # sample F of block k - 1 is sample 0 of block k
        prev_last = bn[F]


def test_fold_phase_rejects_bad_arguments():
    for args in ((0.0, 0.0, 1e8, 64, 0), (-1.0, 0.0, 1e8, 64, 0), (float("nan"), 0.0, 1e8, 64, 0),
                 (1.0, float("inf"), 1e8, 64, 0), (1.0, 0.0, 0.0, 64, 0), (1.0, 0.0, 1e8, 0, 0)):
        with pytest.raises(srtb_b200.SrtbError):
            srtb_b200.fold_phase(*args)


def test_host_pieces(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "fold.mk", "test_fold"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_fold"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "fold ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_executable_rejects_bad_fold_settings(tmp_path):
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "in.bin"
    inp.write_bytes(b"\0" * 4096)
    base = ["--config_file_name", str(tmp_path / "none.cfg"), "--baseband_input_count", "65536",
            "--spectrum_channel_count", "64", "--baseband_sample_rate", "1e8"]
    f = ["--input_file_path", str(inp)]
    for extra, words in ((f + ["--fold_period", "-1"], ["fold_period", "positive"]),
                         (f + ["--fold_period", "1e-6"], ["fold_period", "two spectrum samples"]),
                         (f + ["--fold_period", "0.1", "--fold_bin_count", "5000"], ["fold_bin_count"]),
                         (f + ["--fold_period", "0.1", "--fold_subband_count", "5"], ["fold_subband_count"]),
                         (f + ["--fold_period", "0.1", "--dm_list", "1,2"], ["fold_period", "dm_list"]),
                         (["--fold_period", "0.1"], ["fold_period", "input_file_path"])):
        r = subprocess.run([str(exe), *base, *extra], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, (extra, r.returncode, r.stderr[-2000:])
        assert all(w in r.stderr for w in words), (extra, r.stderr[-2000:])
