"""Host side of the block path's candidates (signal_detect_candidates): the key parsed from a .cfg and from the command
line, its start-up refusal together with either DM search, and the new C entries exported and bound."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import pytest

import srtb_b200 as sb

ROOT = Path(__file__).resolve().parent.parent


def test_entries_are_exported_and_bound():
    lib = sb.load_library()
    for name in ("srtb_b200_submit_block_events", "srtb_b200_collect_block_events"):
        assert name in sb.SYMBOLS
        assert getattr(lib, name).argtypes == sb.SYMBOLS[name][1]
    assert sb.RING_SLOTS == 3
    assert C.sizeof(sb.Event) == 40


def _exe():
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    return str(ROOT / "src" / "srtb_b200")


@pytest.mark.parametrize("search", ["dm_list", "incoherent_dm_list"])
def test_executable_refuses_the_key_with_a_dm_search(tmp_path, search):
    """src/srtb_b200 refuses signal_detect_candidates with either DM search at start-up, from the command line or a
    .cfg, naming the keys (the check runs before any device is touched)"""
    exe = _exe()
    cfg = tmp_path / "k.cfg"
    cfg.write_text(f"signal_detect_candidates = 1\n{search} = 1, 2, 3\n")
    for args in (["--signal_detect_candidates", "1", f"--{search}", "1,2,3"], ["--config_file_name", str(cfg)],
                 ["--signal_detect_candidates", "2 - 1", f"--{search}", "5"]):
        r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=60, cwd=tmp_path)
        assert r.returncode == 2, (args, r.stderr[-2000:])
        msg = r.stderr.strip().splitlines()[-1]
        for key in ("signal_detect_candidates", "dm_list", "incoherent_dm_list", "dm_search_candidates"):
            assert key in msg, (args, msg)


def test_executable_knows_the_key(tmp_path):
    """the key is a known option: an unknown one is refused by name, this one reaches the DM-search refusal instead"""
    exe = _exe()
    r = subprocess.run([exe, "--signal_detect_candidatez", "1"], capture_output=True, text=True, timeout=60,
                       cwd=tmp_path)
    assert r.returncode != 0 and "signal_detect_candidatez" in r.stderr
    r = subprocess.run([exe, "--signal_detect_candidates", "1", "--dm_list", "1"], capture_output=True, text=True,
                       timeout=60, cwd=tmp_path)
    assert r.returncode == 2 and "signal_detect_candidates" in r.stderr
