"""The executable's candidate_cutouts end to end: a recording with pulses dispersed at dm through the block path
(signal_detect_candidates, one stream, and two streams with the total intensity) and through the incoherent search
(incoherent_dm_list + dm_search_candidates). Each candidate file gets its cut-out files: their shapes, the csv's rows
and columns, ft and dmt recomputed by the float64 oracle from the .npy spectrum the executable writes for the block
within the fp32 bound, and the brightest candidate's plane peaking near its centre row and bin. With the key at 0 the
output directory holds the same files as a run without it."""
import numpy as np
import pytest

pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import cutout_oracle as co  # noqa: E402
from test_gpu_block_candidates import (ROOT, X_BW, X_C, X_DM, X_FLOW, X_FS, _outputs, _rows, _x_geometry,  # noqa: E402
                                       _x_recording, _x_run)

W = ROWS = 256
CSV_HEAD = "candidate,center,decimation,time,dm_row_low,dm_row_high"


def _check_block(d, stem, sid, streams, reserved, n_max=4):
    """the cut-outs beside <stem>.<sid>.candidates.csv, recomputed from the block's spectra <stem>.<s>.npy"""
    cand = _rows([d / f"{stem}.{sid}.candidates.csv"])
    ft = np.load(d / f"{stem}.{sid}.cutout_ft.npy")
    dmt = np.load(d / f"{stem}.{sid}.cutout_dmt.npy")
    lines = (d / f"{stem}.{sid}.cutouts.csv").read_text().splitlines()
    assert lines[0] == CSV_HEAD
    rows = [dict(zip(CSV_HEAD.split(","), ln.split(","))) for ln in lines[1:]]
    n = min(n_max, len(cand))
    nsub = X_C  # the largest divisor of C = 256 up to 256
    assert ft.dtype == np.float32 and ft.shape == (n, nsub, W) and dmt.shape == (n, ROWS, W) and len(rows) == n
    # the n highest S/N, highest first, ties in file order
    order = sorted(range(len(cand)), key=lambda i: -float(cand[i]["snr"]))[:n]
    assert [int(r["candidate"]) for r in rows] == order
    spectra = [np.load(d / f"{stem}.{s}.npy") for s in streams]
    P = co.power(spectra, reserved)
    k = co.k_table(X_C, X_FLOW, X_BW, X_FS)
    k_max = float(np.abs(k).max())
    for j, r in enumerate(rows):
        c = cand[int(r["candidate"])]
        b = int(c["boxcar_length"])
        q = max(1, b // 2)
        center = int(c["sample"]) + b // 2
        assert int(r["decimation"]) == q and int(r["center"]) == center
        hw = float(np.float32(W // 2 * q / k_max))
        eft, edmt, erdm = co.cutout(P, k, X_DM, center, float(c["dm"]), hw, q, W, nsub, ROWS)
        assert np.float32(r["dm_row_low"]) == erdm[0] and np.float32(r["dm_row_high"]) == erdm[-1]
        t_bin0 = (float(c["time"]) * X_FS - 2 * X_C * int(c["sample"]) + 2 * X_C * (center - W // 2 * q)) / X_FS
        assert abs(float(r["time"]) - t_bin0) <= 1e-9 * max(1.0, abs(t_bin0))
        S = len(streams)
        for got, want, ch in ((ft[j], eft, X_C // nsub), (dmt[j], edmt, X_C)):
            err = np.abs(got.astype(np.float64) - want)
            assert np.all(err <= co.bound(S, ch, q) * want + 1e-30), (stem, sid, j)
    # the brightest candidate (a pulse at dm): the plane peaks near its centre row and bin
    rr, ii = np.unravel_index(np.argmax(dmt[0]), dmt[0].shape)
    assert abs(rr - ROWS // 2) <= 8 and abs(ii - W // 2) <= 8, (stem, sid, rr, ii)
    return n


def _stems(d, sid):
    return sorted(p.name[:-len(f".{sid}.candidates.csv")] for p in d.glob(f"out_*.{sid}.candidates.csv"))


def _cutout_files(d):
    return sorted(p.name for p in d.iterdir() if "cutout" in p.name)


def test_block_path_single_stream(tmp_path):
    R, L, Lp, share = _x_geometry()
    raw, _ = _x_recording(1, 21)
    d = _x_run(tmp_path, "on", raw, "simple", ["--signal_detect_candidates", "1", "--candidate_cutouts", "4"])
    total = 0
    for stem in _stems(d, "0"):
        if _rows([d / f"{stem}.0.candidates.csv"]):
            total += _check_block(d, stem, "0", [0], L - Lp)
        else:
            assert not (d / f"{stem}.0.cutouts.csv").exists()
    assert total >= 3


def test_block_path_two_streams_and_the_sum(tmp_path):
    R, L, Lp, share = _x_geometry()
    raw, _ = _x_recording(2, 22)
    d = _x_run(tmp_path, "on", raw, "naocpsr_snap1", ["--signal_detect_candidates", "1",
                                                      "--signal_detect_sum_polarizations", "1",
                                                      "--candidate_cutouts", "4"])
    seen = {"0": 0, "1": 0, "sum": 0}
    for sid, streams in (("0", [0]), ("1", [1]), ("sum", [0, 1])):
        for stem in _stems(d, sid):
            if _rows([d / f"{stem}.{sid}.candidates.csv"]):
                seen[sid] += _check_block(d, stem, sid, streams, L - Lp)
    assert all(v >= 3 for v in seen.values()), seen


def test_incoherent_search(tmp_path):
    R, L, Lp, share = _x_geometry()
    raw, _ = _x_recording(1, 23)
    d = _x_run(tmp_path, "on", raw, "simple", ["--incoherent_dm_list", f"{X_DM - 0.3}:{X_DM + 0.3}:0.05",
                                               "--dm_search_candidates", "1", "--candidate_cutouts", "4"])
    total = 0
    for stem in _stems(d, "0"):
        if _rows([d / f"{stem}.0.candidates.csv"]):
            total += _check_block(d, stem, "0", [0], L - Lp)
    assert total >= 3


def test_key_at_zero_writes_todays_files(tmp_path):
    raw, _ = _x_recording(2, 24)
    base = ["--signal_detect_candidates", "1", "--signal_detect_sum_polarizations", "1"]
    off = _x_run(tmp_path, "off", raw, "naocpsr_snap1", base)
    zero = _x_run(tmp_path, "zero", raw, "naocpsr_snap1", base + ["--candidate_cutouts", "0"])
    a, b = _outputs(off), _outputs(zero)
    assert a and [n for n, _ in a] == [n for n, _ in b] and a == b
    assert not _cutout_files(off) and not _cutout_files(zero)
