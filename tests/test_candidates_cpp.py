"""CPU checks of the DM search candidates' host pieces (tests/cpp/test_candidates.cpp): the dm_search_candidates key in
a .cfg and on the command line, its start-up check, and the exact candidates.csv text write_signal_pipe writes."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_cpp_candidates(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "candidates.mk", "test_candidates"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_candidates"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "candidates ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
