"""CPU checks of the incoherent DM search's trial grouping: srtb_b200_incoherent_groups (the grouping the search launches
with) against its restatement in tests/incoherent_grouping.py, and every case of tests/incoherent_cases.py reaching the
grouping, spread and T-residue structure its GPU test (tests/test_gpu_incoherent_geometry.py) is named for."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

import incoherent_cases as ic
import incoherent_grouping as ig
import incoherent_oracle as io
import srtb_b200

CASES = ic.cases()


def _structure(case):
    fl, bw = ic.BANDS[case["band"]]
    s, sp, sm = io.shifts(ic.C, fl, bw, ic.SR, ic.DM, case["dms"])
    order, groups, gmin, gmax, spread = ig.groups(s, case["dms"])
    T = case["time_count"] - case["reserved"] - sp - sm
    return s, sm, order, groups, gmin, gmax, spread, T


def _cut(s, order, groups, i):
    """why group i ends: "count" (64 trials; the next one would fit the spread), "spread" (the next trial would push
    some channel over INC_SPREAD_MAX) or "end" (the list ends)"""
    first, count = groups[i]
    if first + count == len(order):
        return "end"
    rows = s[order[first:first + count + 1]]
    fits = int((rows.max(0) - rows.min(0)).max()) <= ig.INC_SPREAD_MAX
    if count == ig.INC_GROUP:
        return "count" if fits else "count+spread"
    assert not fits
    return "spread"


@pytest.mark.parametrize("name", sorted(CASES))
def test_library_groups_match_restatement(name):
    case = CASES[name]
    fl, bw = ic.BANDS[case["band"]]
    s, sm, order, groups, gmin, gmax, spread, _ = _structure(case)
    g_order, g_groups, g_gspan, g_spread = srtb_b200.incoherent_groups(ic.C, fl, bw, ic.SR, ic.DM, case["dms"])
    assert np.array_equal(g_order, order)
    assert [tuple(g) for g in g_groups] == groups
    assert np.array_equal(g_gspan[:, :, 0], gmin + sm) and np.array_equal(g_gspan[:, :, 1], gmax + sm)
    assert g_spread == spread


def test_grouping_restatement_on_a_known_answer():
    """hand-made shifts: a spread of exactly INC_SPREAD_MAX fits, one more does not; 64 trials fill a group"""
    s = np.array([[0, 0], [1792, 5], [1793, 0], [1793, 1]])
    order, groups, gmin, gmax, spread = ig.groups(s, [0.0, 1.0, 2.0, 3.0])
    assert groups == [(0, 2), (2, 2)] and spread == 1792
    assert np.array_equal(gmin, [[0, 0], [1793, 0]]) and np.array_equal(gmax, [[1792, 5], [1793, 1]])
    order, groups, _, _, spread = ig.groups(np.zeros((130, 3), np.int64), [1.0] * 130)
    assert groups == [(0, 64), (64, 64), (128, 2)] and spread == 0 and np.array_equal(order, np.arange(130))
    order, _, _, _, _ = ig.groups(np.zeros((4, 1), np.int64), [2.0, 1.0, 2.0, 1.0])
    assert list(order) == [1, 3, 0, 2]  # stable


@pytest.mark.parametrize("name", ["upright", "inverted"])
def test_geometry_cases_are_cut_by_count_and_by_spread(name):
    s, _, order, groups, _, _, _, T = _structure(CASES[name])
    cuts = [_cut(s, order, groups, i) for i in range(len(groups))]
    # a spread-cut group spans 1792 samples at the band edge, 0.6 DM on the inverted band: one such cut fits under 1 DM
    assert "count" in cuts and cuts.count("spread") >= (2 if name == "upright" else 1), cuts
    assert 100 <= len(CASES[name]["dms"]) <= 250
    assert ic.DM in CASES[name]["dms"]
    dms = np.asarray(CASES[name]["dms"], np.float64)
    if name == "inverted":
        assert dms.max() - dms.min() < 1.0
    else:
        assert dms.max() - dms.min() > 3.0
        # a run of single-trial groups: neighbours more than INC_SPREAD_MAX apart at the band edge
        counts = [c for _, c in groups]
        assert counts[-3:] == [1, 1, 1], counts
        srt = s[order]
        assert all(np.abs(srt[i] - srt[i - 1]).max() > ig.INC_SPREAD_MAX for i in range(len(order) - 3, len(order)))
    assert T > 4000


def test_spread_1792_case_fits_exactly_and_the_next_trial_does_not():
    s, _, order, groups, gmin, gmax, spread, _ = _structure(CASES["spread_1792"])
    first, count = groups[0]
    assert int((gmax[0] - gmin[0]).max()) == ig.INC_SPREAD_MAX == 1792
    rows = s[order[first:first + count + 1]]
    assert int((rows.max(0) - rows.min(0)).max()) == 1793
    assert count < ig.INC_GROUP and len(groups) == 2 and spread == 1792


@pytest.mark.parametrize("name,spread,opt_in", [("smem_1472", 1472, False), ("smem_1473", 1473, True)])
def test_shared_memory_cases_straddle_48_kib(name, spread, opt_in):
    *_, got, _ = _structure(CASES[name])
    assert got == spread
    assert (ig.smem_bytes(got) > 48 * 1024) == opt_in
    assert ig.smem_bytes(1472) == 48 * 1024


def test_order_cases_permute_the_upright_list():
    up = CASES["upright"]["dms"]
    sh, rv, dup = CASES["shuffled"]["dms"], CASES["reversed"]["dms"], CASES["duplicates"]["dms"]
    assert sorted(sh) == sorted(up) and sh != up and sh != sorted(sh)
    assert rv == up[::-1]
    assert len(set(dup)) == len(set(up)) < len(dup)
    # the stable sort keeps duplicates in list order, and the groups are the upright list's with the copies inside
    _, _, order, groups, _, _, _, _ = _structure(CASES["duplicates"])
    srt = np.asarray(dup, np.float32)[order]
    assert np.all(np.diff(srt) >= 0)
    for i in range(len(order) - 1):
        if srt[i] == srt[i + 1]:
            assert order[i] < order[i + 1]
    for name in ("shuffled", "reversed"):
        a = _structure(CASES[name])
        b = _structure(CASES["upright"])
        assert a[3] == b[3] and np.array_equal(np.asarray(CASES[name]["dms"])[a[2]], np.asarray(up)[b[2]])


@pytest.mark.parametrize("name,residue", [("upright", 0), ("tail_1", 1), ("tail_255", 255)])
def test_series_length_residues(name, residue):
    *_, T = _structure(CASES[name])
    assert T % ig.INC_TILE == residue and T > ig.INC_TILE
    if name.startswith("tail"):
        assert CASES[name]["reserved"] == 0
        _, _, order, groups, _, _, _, _ = _structure(CASES[name])
        assert len(groups) >= 2


def test_short_series_is_one_partial_tile():
    *_, T = _structure(CASES["short"])
    assert 2 <= T < ig.INC_TILE


def test_long_series_pass_gridDim_y():
    _, sp, sm = io.shifts(ic.LONG_C, *ic.LONG_BAND, ic.LONG_SR, ic.DM, ic.LONG_DMS)
    assert sp > 0 and sm > 0 and sp + sm == ic.long_span()
    tiles = {k: -(-T // ig.INC_TILE) for k, T in ic.LONG_T.items()}
    assert tiles["65535_tiles"] == 65535 and tiles["65535_tiles_plus_1"] == 65536
    assert ic.LONG_T["2^24+2^17"] > 65535 * 256 and ic.LONG_T["2^24+2^17"] + sp + sm < (1 << 30)


def test_groups_entry_refuses_bad_arguments():
    lib = srtb_b200.load_library()
    arr = (C.c_float * 2)(100.0, 100.001)  # 72 samples apart at the edge: one group
    ng = C.c_uint64()
    E_INVALID = -1
    assert lib.srtb_b200_incoherent_groups(0, 1000.0, 500.0, 1e9, 100.0, arr, 2, None, None, None, C.byref(ng),
                                           None) == E_INVALID
    assert lib.srtb_b200_incoherent_groups(16, 1000.0, 500.0, 1e9, 100.0, None, 2, None, None, None, C.byref(ng),
                                           None) == E_INVALID
    assert lib.srtb_b200_incoherent_groups(16, 1000.0, 500.0, 1e9, 100.0, arr, 0, None, None, None, C.byref(ng),
                                           None) == E_INVALID
    assert lib.srtb_b200_incoherent_groups(16, 1000.0, 500.0, 1e9, 100.0, arr, 2, None, None, None, None,
                                           None) == E_INVALID
    assert lib.srtb_b200_incoherent_groups(16, 1000.0, 500.0, 1e9, 100.0, arr, 2, None, None, None, C.byref(ng),
                                           None) == 0 and ng.value == 1


def test_groups_entry_is_exported_and_bound():
    out = subprocess.run(["nm", "-D", "--defined-only", str(srtb_b200.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    assert re.search(r"\bT srtb_b200_incoherent_groups\b", out)
    assert "srtb_b200_incoherent_groups" in srtb_b200.SYMBOLS
