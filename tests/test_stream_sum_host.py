"""CPU checks of the total-intensity detector's host pieces: the signal_detect_sum_polarizations key, its start-up
rejections and the sink's keep rule and .sum.<boxcar>.tim files (tests/cpp/test_stream_sum.cpp), and the binding's
block-config field."""
import ctypes as C
import subprocess
from pathlib import Path

import srtb_b200

ROOT = Path(__file__).resolve().parent.parent


def test_host_pieces(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "stream_sum.mk", "test_stream_sum"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_stream_sum"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "stream_sum ok" in r.stdout, r.stderr[-2000:]


def test_block_config_field_is_last_and_off_by_default():
    cfg = srtb_b200.BlockConfig()
    assert cfg.signal_detect_sum_streams == 0
    names = [f[0] for f in srtb_b200.BlockConfig._fields_]
    assert names[-1] == "signal_detect_sum_streams"
    assert srtb_b200.BlockConfig.signal_detect_sum_streams.offset == \
        srtb_b200.BlockConfig.n_rfi_freq_pairs.offset + C.sizeof(C.c_uint64)


def test_executable_rejects_sum_with_one_stream(tmp_path):
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    for extra, word in ((["--baseband_format_type", "simple"], "two or more streams"),
                        (["--baseband_format_type", "naocpsr_snap1", "--dm_list", "1,2"], "dm_list"),
                        (["--baseband_format_type", "naocpsr_snap1", "--incoherent_dm_list", "1,2"],
                         "incoherent_dm_list")):
        r = subprocess.run([str(exe), "--config_file_name", str(tmp_path / "none.cfg"),
                            "--signal_detect_sum_polarizations", "1", *extra], capture_output=True, text=True,
                           timeout=60)
        assert r.returncode == 2, (extra, r.returncode, r.stderr[-2000:])
        assert "signal_detect_sum_polarizations" in r.stderr and word in r.stderr, r.stderr[-2000:]
