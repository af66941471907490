"""srtb_b200_correlator's integrating mode (--segment_size) refuses bad options, bad segment sizes and files without a
complete segment from the file sizes alone, before it reads a byte or touches a device; and the library exports the
two entries of that mode. No GPU (the accepted runs are in tests/test_gpu_correlator_segments.py)."""
import os
import re
import subprocess
from pathlib import Path

import pytest

import srtb_b200

ROOT = Path(__file__).resolve().parent.parent
EXE = ROOT / "src" / "srtb_b200_correlator"


def _run(args, cwd):
    if not EXE.exists():
        pytest.fail(f"{EXE} is not built (make -C src)")
    return subprocess.run([str(EXE), *args], cwd=cwd, capture_output=True, text=True, timeout=60)


def _files(tmp_path, s1, s2):
    for name, size in (("a.bin", s1), ("b.bin", s2)):
        with open(tmp_path / name, "wb") as f:
            os.truncate(f.fileno(), size)  # sparse: nothing is written, and nothing must be read
    return ["--input_file_1", str(tmp_path / "a.bin"), "--input_file_2", str(tmp_path / "b.bin"),
            "--output_file", str(tmp_path / "corr.bin")]


@pytest.mark.parametrize("bits", ["1", "2", "4", "-8"])
def test_input_bits_needs_segment_size(tmp_path, bits):
    r = _run(_files(tmp_path, 1 << 12, 1 << 12) + ["--input_bits", bits], tmp_path)
    assert r.returncode == 2 and "usage" in r.stderr and "--segment_size" in r.stderr, r.stderr
    assert not (tmp_path / "corr.bin").exists()


@pytest.mark.parametrize("args", [["--input_bits", "3"], ["--input_bits", "16"], ["--input_bits", "-4"],
                                  ["--input_bits", "x"], ["--segment_size", "x"], ["--segment_size", "-16"],
                                  ["--segment_size", ""], ["--segment_size"]])
def test_bad_segment_options(tmp_path, args):
    r = _run(args, tmp_path)
    assert r.returncode == 2 and "usage" in r.stderr, r.stderr


@pytest.mark.parametrize("ls", [0, 8, 1000, 4097, 1 << 31])
def test_refuses_segment_size_before_reading(tmp_path, ls):
    """with the library's message, on 16 GiB sparse files"""
    r = _run(_files(tmp_path, 1 << 34, 1 << 34) + ["--segment_size", str(ls)], tmp_path)
    assert r.returncode == 1, r.stderr
    assert f"segment_size must be a power of two from 16 to 2^30, got {ls}" in r.stderr
    assert not (tmp_path / "corr.bin").exists()


@pytest.mark.parametrize("s1, s2, bits, ls, samples", [
    (4095, 1 << 34, "8", 4096, "4095 and 17179869184"),
    (1 << 34, 1023, "2", 4096, "68719476736 and 4092"),
    (1 << 20, 1 << 20, "1", 1 << 24, "8388608 and 8388608"),
    (7, 7, "4", 16, "14 and 14"),
    (0, 0, "-8", 16, "0 and 0"),
])
def test_refuses_no_complete_segment_before_reading(tmp_path, s1, s2, bits, ls, samples):
    r = _run(_files(tmp_path, s1, s2) + ["--segment_size", str(ls), "--input_bits", bits], tmp_path)
    assert r.returncode == 1, r.stderr
    assert f"no complete segment of {ls} samples: {samples} samples" in r.stderr
    assert not (tmp_path / "corr.bin").exists()


def test_segment_entries_are_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", str(srtb_b200.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    exported = set(re.findall(r"\bT (srtb_b200_[a-z0-9_]+)", out))
    for name in ("srtb_b200_correlate_accumulate", "srtb_b200_correlate_finish"):
        assert name in exported and name in srtb_b200.SYMBOLS
    header = (ROOT / "include" / "srtb_b200.h").read_text()
    assert "int srtb_b200_correlate_accumulate(" in header and "int srtb_b200_correlate_finish(" in header
