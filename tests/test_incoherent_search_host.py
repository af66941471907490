"""CPU checks of the incoherent DM search's host pieces: srtb_b200_incoherent_shifts against the float64 oracle
(tests/incoherent_oracle.py) for both band orientations, trials on both sides of dm and exact half-sample ties; the
oracle's own known answer; the incoherent_dm_list key, its conflict with dm_list, the block overlap and the reader's
offsets (tests/cpp/test_incoherent.cpp); and the exported entries."""
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import incoherent_oracle as io
import srtb_b200

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.parametrize("f_low,bw", [(1000.0, 500.0), (1500.0, -500.0), (1437.0, -64.0)])
@pytest.mark.parametrize("C_", [1, 16, 2048])
def test_shifts_match_oracle(f_low, bw, C_):
    dm = 56.778
    dms = [dm - 0.7, dm - 0.013, dm, dm + 0.0041, dm + 1.3, 0.0, 2 * dm]
    got, sp, sm = srtb_b200.incoherent_shifts(C_, f_low, bw, 1e9, dm, dms)
    want, wsp, wsm = io.shifts(C_, f_low, bw, 1e9, dm, dms)
    assert np.array_equal(got, want)
    assert (sp, sm) == (wsp, wsm)
    assert not got[2].any()  # the trial at dm
    # channel 0 is the farthest from f_ref in both orientations. Below f_ref (bw > 0) a larger DM arrives later there,
    # so its shift is positive; above f_ref (bw < 0, f_ref = the bottom edge) it arrives earlier: negative
    if C_ > 1:
        sign = 1 if bw > 0 else -1
        assert sign * got[4, 0] > 0 > sign * got[0, 0]
    _, sp2, sm2 = srtb_b200.incoherent_shifts(C_, f_low, bw, 1e9, dm, dms, table=False)
    assert (sp2, sm2) == (sp, sm)


def _find_tie(C_, f_low, bw, sr):
    """(DM_d, dm, channel, n): float32 values whose unrounded shift is exactly n + 0.5 in the library's arithmetic"""
    k = io.shift_values(C_, f_low, bw, sr, 0.0, [1.0])[0]
    for n in range(1, 4000):
        for c in range(C_):
            if k[c] <= 0:
                continue
            t = n + 0.5
            dmd = np.float32(t / k[c])
            resid = (float(dmd) * k[c] - t) / k[c]
            for dm in (np.float32(resid), np.nextafter(np.float32(resid), np.float32(1)),
                       np.nextafter(np.float32(resid), np.float32(-1))):
                if io.shift_values(C_, f_low, bw, sr, float(dm), [float(dmd)])[0][c] == t:
                    return float(dmd), float(dm), c, n
    raise AssertionError("no exact tie found")


def test_half_sample_tie_rounds_away_from_zero():
    C_, f_low, bw, sr = 8, 1000.0, 500.0, 1e8
    dmd, dm, c, n = _find_tie(C_, f_low, bw, sr)
    got, _, _ = srtb_b200.incoherent_shifts(C_, f_low, bw, sr, dm, [dmd])
    want, _, _ = io.shifts(C_, f_low, bw, sr, dm, [dmd])
    assert np.array_equal(got, want)
    assert got[0, c] == n + 1  # llround: n + 0.5 -> n + 1
    # the mirrored trial: -(n + 0.5) -> -(n + 1)
    got_neg, _, sm = srtb_b200.incoherent_shifts(C_, f_low, bw, sr, -dm, [-dmd])
    assert got_neg[0, c] == -(n + 1) and sm >= n + 1
    assert np.array_equal(got_neg, io.shifts(C_, f_low, bw, sr, -dm, [-dmd])[0])


def test_oracle_impulses_along_one_trial_sum_to_C_there_only():
    """one unit impulse per channel on trial k's curve: v_k peaks at C at that time, every other trial stays below"""
    C_, L, f_low, bw, sr, dm = 32, 2048, 1000.0, 500.0, 1e8, 10.0
    dms = [dm + 0.05 * i for i in range(-4, 5)]
    s, sp, sm = io.shifts(C_, f_low, bw, sr, dm, dms)
    for k in range(len(dms)):
        x = np.zeros((C_, L), np.complex64)
        x[:, 0] = 1e-3  # a non-zero first sample: no channel counts as flagged
        j0 = 300
        for c in range(C_):
            x[c, j0 + sm + s[k, c]] = 1.0
        v = io.series(np.abs(x.astype(np.complex128)) ** 2, L, s, sp, sm)
        assert v[k, j0] == C_ and np.delete(v[k], j0).max() < 1
        others = np.delete(v, k, axis=0)
        assert others.max() < C_
        # on the unsmoothed series (boxcar 1) trial k has the largest peak S/N, at j0
        trials, _, _ = io.search(x, 0, f_low, bw, sr, dm, dms, 6.0, 0.9, 16)
        assert int(np.argmax([t["peak_snr"][0] for t in trials])) == k and trials[k]["peak_index"][0] == j0


def test_cpp_incoherent(tmp_path):
    d = ROOT / "tests" / "cpp"
    subprocess.run(["make", "-C", str(d), "-f", "incoherent.mk", "test_incoherent"], check=True, capture_output=True)
    r = subprocess.run([str(d / "test_incoherent"), str(tmp_path)], capture_output=True, text=True, timeout=120,
                       env={"SRTB_LOG_LEVEL": "1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "incoherent ok" in r.stdout, r.stderr[-2000:]


def test_incoherent_entries_are_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", str(srtb_b200.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    for name in ("srtb_b200_incoherent_shifts", "srtb_b200_incoherent_dm_search"):
        assert re.search(rf"\bT {name}\b", out), name
        assert name in srtb_b200.SYMBOLS
    srtb_b200.load_library()
