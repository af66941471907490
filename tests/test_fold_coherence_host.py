"""CPU checks of the folded coherence products' host pieces: the fold_coherence key, its start-up rejections, the sink's
coherence accumulator (tests/cpp/test_fold_coherence.cpp), and the executable's rejections."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_host_pieces(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "fold_coherence.mk", "test_fold_coherence"], check=True,
                   capture_output=True)
    r = subprocess.run([str(d / "test_fold_coherence"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "fold coherence ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_executable_rejects_bad_coherence_settings(tmp_path):
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "in.bin"
    inp.write_bytes(b"\0" * 4096)
    base = ["--config_file_name", str(tmp_path / "none.cfg"), "--baseband_input_count", "65536",
            "--spectrum_channel_count", "64", "--baseband_sample_rate", "1e8", "--input_file_path", str(inp)]
    fold = ["--fold_period", "0.1", "--fold_coherence", "1"]
    for extra, words in ((["--fold_coherence", "1", "--baseband_format_type", "naocpsr_snap1"],
                          ["fold_coherence", "fold_period"]),
                         (fold + ["--baseband_format_type", "simple"], ["fold_coherence", "single-stream"]),
                         (fold + ["--baseband_format_type", "fastmb_roach2"], ["fold_coherence", "single-stream"]),
                         (fold + ["--baseband_format_type", "gznupsr_a1_4"], ["fold_coherence", "gznupsr_a1_4"])):
        r = subprocess.run([str(exe), *base, *extra], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, (extra, r.returncode, r.stderr[-2000:])
        assert all(w in r.stderr for w in words), (extra, r.stderr[-2000:])
