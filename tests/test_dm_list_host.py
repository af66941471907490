"""CPU checks of the DM search's host pieces (tests/cpp/test_dm_list.cpp): the dm_list config key, the block overlap a
DM list needs in read_file_pipe, the candidate files write_signal_pipe writes for a sweep, and the exported entry."""
import re
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_cpp_dm_list(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "dm_list.mk", "test_dm_list"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_dm_list"), str(tmp_path), str(ROOT / "tests" / "golden")], capture_output=True,
                       text=True, timeout=120, env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "dm list ok" in r.stdout, r.stderr[-2000:]


def test_dm_sweep_ex_is_exported():
    import srtb_b200
    out = subprocess.run(["nm", "-D", "--defined-only", str(srtb_b200.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    assert re.search(r"\bT srtb_b200_process_block_dm_sweep_ex\b", out)
    assert "srtb_b200_process_block_dm_sweep_ex" in srtb_b200.SYMBOLS
    srtb_b200.load_library()  # binds it with the declared argument types
