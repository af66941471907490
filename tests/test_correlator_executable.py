"""srtb_b200_correlator refuses what srtb_b200_correlate would refuse from the file sizes alone, before it reads a byte
or touches a device, with a message and a non-zero exit status; and bad options. No GPU (the accepted runs are in
tests/test_gpu_correlator.py)."""
import os
import subprocess
from pathlib import Path

import pytest

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


@pytest.mark.parametrize("s1, s2, text", [
    (1 << 32, 1 << 32, "above 2^31"),
    ((1 << 33) + 1, (1 << 32) + 1, "above 2^31"),
    (3000, 1 << 20, "[fft] n must be a power of 2, got 3000"),
    (1 << 12, 6, "[fft] n must be a power of 2, got 6"),
    (1, 1 << 12, "at least 2 bytes"),
    (0, 0, "at least 2 bytes"),
])
def test_refuses_sizes_before_reading(tmp_path, s1, s2, text):
    r = _run(_files(tmp_path, s1, s2), tmp_path)
    assert r.returncode == 1, r.stderr
    assert text in r.stderr
    assert not (tmp_path / "corr.bin").exists()


def test_missing_input_uses_the_default_names(tmp_path):
    """no options: pol_1.bin and pol_2.bin in the working directory, as in the reference"""
    r = _run([], tmp_path)
    assert r.returncode == 1 and "pol_1.bin" in r.stderr, r.stderr
    (tmp_path / "pol_1.bin").write_bytes(b"\0" * 16)
    r = _run([], tmp_path)
    assert r.returncode == 1 and "pol_2.bin" in r.stderr, r.stderr


@pytest.mark.parametrize("args", [["--bogus", "1"], ["--gpu_device", "x"], ["--gpu_device", "-1"], ["--output_file"]])
def test_bad_options(tmp_path, args):
    r = _run(args, tmp_path)
    assert r.returncode == 2 and "usage" in r.stderr, r.stderr
