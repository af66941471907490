"""Host side of the candidate cut-outs: the float64 oracle's known answers (an impulse lands in its predicted bin at
every decimation; a pulse dispersed at dm + delta peaks at delta's row and bin W/2), its shift table against the
incoherent search's, the C entry exported and bound, the candidate_cutouts key and its start-up refusals in the
executable, and the C++ host pieces (tests/cpp/test_cutouts.cpp: the key, the top-N selection, the half-width rule and
the exact cutouts.csv text)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import cutout_oracle as co
import incoherent_oracle as io
import srtb_b200 as sb

ROOT = Path(__file__).resolve().parent.parent
SR = 2e8


def test_shift_table_at_q1_is_the_incoherent_searchs():
    for fl, bw in ((1000.0, 200.0), (1200.0, -300.0)):
        dms = [29.0, 30.0, 30.37, 31.5, 45.0]
        k = co.k_table(64, fl, bw, SR)
        s, _, _ = io.shifts(64, fl, bw, SR, 30.0, dms)
        assert np.array_equal(co.shifts(k, 30.0, dms, 1), s)
        lib_s, _, _ = sb.incoherent_shifts(64, fl, bw, SR, 30.0, dms)
        assert np.array_equal(co.shifts(k, 30.0, dms, 1), lib_s)


def test_row_dms():
    assert co.row_dms(5.0, 1.0, 1).tolist() == [5.0]
    r = co.row_dms(5.0, 1.0, 256)
    assert r[128] == np.float32(5.0) and r[0] == np.float32(4.0) and np.all(np.diff(r) > 0)
    r = co.row_dms(5.0, 2.0, 255)
    assert r[127] == np.float32(5.0) and r[0] == np.float32(3.0) and r[254] == np.float32(7.0)


@pytest.mark.parametrize("q", [1, 3, 16, 128])
def test_impulse_lands_in_its_bin(q):
    """one sample of one channel: in the image at q = 1 and nsub = C it sits at bin (j - t0) / q - s of that channel;
    every other bin and channel is 0"""
    C, L, W = 16, 1 << 16, 128
    fl, bw, dm = 1000.0, 100.0, 3.0
    x = np.zeros((C, L), np.complex64)
    x[:, 0] = 1e-3  # every channel kept
    c0, j = 5, 20000 + 7
    x[c0, j] = 2.0
    center, d_req = 20000, 3.003
    ft, dmt, _ = co.cutouts([x], 0, fl, bw, SR, dm, [(center, d_req, 0.5, q)], W, C, 5)
    s = co.shifts(co.k_table(C, fl, bw, SR), dm, [d_req], q)[0]
    t0 = center - (W // 2) * q
    b = (j - t0) // q - s[c0]
    assert 0 <= b < W
    img = ft[0].copy()
    assert img[c0, b] == 4.0
    img[c0, b] = 0
    assert np.count_nonzero(img) == 0
    assert np.all(np.isin(dmt[0], [0.0, 4.0]))


@pytest.mark.parametrize("bw", [200.0, -200.0])
def test_dispersed_pulse_peaks_at_its_row_and_the_centre(bw):
    """a pulse dispersed at dm + delta (residual delays s(dm + delta, c) from bin 0 of the reference) peaks in the plane
    at the row of dm + delta and at bin W/2, and its image at that DM is a straight column at W/2"""
    C, L, W, n_rows = 64, 1 << 15, 128, 65
    fl, dm, delta, q = 1000.0, 40.0, 0.3, 2
    k = co.k_table(C, fl, bw, SR)
    hw = (W / 2) * q / np.abs(k).max()
    dms = co.row_dms(dm, hw, n_rows)
    r_want = int(np.argmin(np.abs(dms - np.float32(dm + delta))))
    d_pulse = float(dms[r_want])
    s = co.shifts(k, dm, [d_pulse], 1)[0]
    t_pulse = 16000
    x = np.zeros((C, L), np.complex64)
    x[:, 0] = 1e-3
    for c in range(C):
        x[c, t_pulse + s[c]: t_pulse + s[c] + q] = 1.0
    ft, dmt, _ = co.cutouts([x], 0, fl, bw, SR, dm, [(t_pulse, dm, hw, q)], W, C, n_rows)
    r, i = np.unravel_index(np.argmax(dmt[0]), dmt[0].shape)
    assert r == r_want and i == W // 2, (r, i, r_want)
    # a channel's q samples fill bin W/2, or straddle it and a neighbour where its shift in decimated bins rounds off
    ft2, _, _ = co.cutouts([x], 0, fl, bw, SR, dm, [(t_pulse, d_pulse, hw, q)], W, C, 1)
    assert np.all(np.isin(np.argmax(ft2[0], axis=1), [W // 2 - 1, W // 2, W // 2 + 1]))
    assert np.all(ft2[0][:, W // 2 - 1:W // 2 + 2].sum(axis=1) == q)


def test_entry_is_exported_and_bound():
    lib = sb.load_library()
    name = "srtb_b200_candidate_cutouts"
    assert name in sb.SYMBOLS and getattr(lib, name).argtypes == sb.SYMBOLS[name][1]
    assert C.sizeof(sb.CutoutRequest) == 24
    assert sb.CutoutRequest.decimation.offset == 16


def test_cpp_cutouts(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "cutouts.mk", "test_cutouts"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_cutouts"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "cutouts ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def _exe():
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    return str(ROOT / "src" / "srtb_b200")


@pytest.mark.parametrize("args, words", [
    (["--candidate_cutouts", "-2", "--signal_detect_candidates", "1"], ["candidate_cutouts", "-2"]),
    (["--candidate_cutouts", "4"], ["candidate_cutouts", "signal_detect_candidates", "dm_search_candidates"]),
    (["--candidate_cutouts", "4", "--dm_search_candidates", "1", "--dm_list", "1,2"], ["candidate_cutouts", "dm_list"]),
])
def test_executable_refuses_at_start_up(tmp_path, args, words):
    """refused from the command line and from a .cfg, before any device is touched, naming the keys"""
    exe = _exe()
    cfg = tmp_path / "k.cfg"
    lines = [f"{a[2:]} = {b}" for a, b in zip(args[::2], args[1::2])]
    cfg.write_text("\n".join(lines) + "\n")
    for argv in (args, ["--config_file_name", str(cfg)]):
        r = subprocess.run([exe] + argv, capture_output=True, text=True, timeout=60, cwd=tmp_path)
        assert r.returncode == 2, (argv, r.stderr[-2000:])
        msg = r.stderr.strip().splitlines()[-1]
        for w in words:
            assert w in msg, (argv, msg)
