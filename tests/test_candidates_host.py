"""Host-side tests of the single-pulse candidate list: srtb_b200_cluster_events against the pairwise union-find
restatement in candidates_oracle.py, its argument checks, and the ctypes mirrors of srtb_b200_event and
srtb_b200_candidate (no GPU needed: clustering runs on the host)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import candidates_oracle as oracle
import srtb_b200 as sb

EV = sb._dtype_of(sb.Event)


def _random_events(rng, n, n_dm, streams, t_max, max_b=8):
    """n events whose runs never overlap within one (stream, trial, boxcar) row, as the device produces them"""
    ev = np.zeros(n, EV)
    rows = {}
    for i in range(n):
        s, d, b = int(rng.integers(streams)), int(rng.integers(n_dm)), int(rng.integers(max_b))
        ev[i]["stream"], ev[i]["trial"], ev[i]["boxcar"] = s, d, b
        ev[i]["snr"] = np.float32(rng.choice([6.5, 7.0, 8.0, 9.5, 12.0]))  # few values: ties for the representative
        rows.setdefault((s, d, b), []).append(i)
    for idx in rows.values():
        starts = np.sort(rng.choice(t_max, size=len(idx), replace=False)) * 4  # spaced: disjoint runs
        for k, i in enumerate(idx):
            length = int(rng.integers(1, 4))
            ev[i]["begin"] = starts[k]
            ev[i]["end"] = starts[k] + length
            ev[i]["peak_index"] = starts[k] + int(rng.integers(length))
    return ev


def _check(ev, dms, max_candidates=None):
    got, total = sb.cluster_events(ev, dms, max_candidates)
    want = oracle.cluster(ev, dms)
    assert total == len(want)
    cap = len(want) if max_candidates is None else max_candidates
    assert len(got) == min(cap, len(want))
    for g, w in zip(got, want):
        for k, v in w.items():
            assert g[k] == v, (k, g[k], v)
    return got, total


@pytest.mark.parametrize("n,n_dm,streams,seed", [(0, 3, 1, 0), (1, 1, 1, 1), (40, 5, 2, 2), (500, 16, 3, 3),
                                                 (5000, 64, 2, 4)])
def test_cluster_matches_oracle(n, n_dm, streams, seed):
    rng = np.random.default_rng(seed)
    dms = rng.uniform(0, 100, n_dm).astype(np.float32)
    if n_dm >= 4:
        dms[1] = dms[3]  # repeated DMs: adjacent ranks
    ev = _random_events(rng, n, n_dm, streams, t_max=max(n // 2, 8))
    _check(ev, dms)


def test_cluster_shuffled_input_and_dms():
    rng = np.random.default_rng(7)
    dms = rng.permutation(np.arange(20, dtype=np.float32))
    ev = _random_events(rng, 800, 20, 2, t_max=300)
    a, _ = _check(ev, dms)
    b, _ = sb.cluster_events(ev[rng.permutation(len(ev))], dms)
    assert a.tobytes() == b.tobytes()


def test_cluster_transitive_chain():
    """a and c are not friends (ranks 2 apart), b joins them: one candidate of three"""
    dms = [10.0, 11.0, 12.0, 50.0]
    ev = np.zeros(4, EV)
    # the last event meets the third in time and rank but is in another stream
    for i, (trial, b0, e0, snr, s) in enumerate([(0, 100, 102, 7.0, 0), (2, 102, 104, 8.0, 0), (1, 101, 103, 9.0, 0),
                                                 (3, 102, 104, 20.0, 1)]):
        ev[i]["trial"], ev[i]["begin"], ev[i]["end"], ev[i]["peak_index"], ev[i]["snr"] = trial, b0, e0, b0, snr
        ev[i]["stream"] = s
    got, total = _check(ev, dms)
    assert total == 2
    c = got[0]
    assert c["members"] == 3 and c["trial"] == 1 and c["dm_low"] == 10.0 and c["dm_high"] == 12.0
    assert (c["span_begin"], c["span_end"]) == (100, 104)
    assert got[1]["members"] == 1 and got[1]["trial"] == 3 and got[1]["stream"] == 1
    ev[2]["begin"], ev[2]["end"], ev[2]["peak_index"] = 300, 301, 300  # without the middle event: apart
    _, total = _check(ev, dms)
    assert total == 4


def test_cluster_span_of_boxcars():
    """b = 0 spans [begin, end); b >= 1 spans [begin + 1, end + 2^b): events that only meet through a boxcar's window"""
    dms = [1.0]
    ev = np.zeros(2, EV)
    ev[0]["begin"], ev[0]["end"], ev[0]["peak_index"], ev[0]["snr"], ev[0]["boxcar"] = 10, 11, 10, 7, 0
    ev[1]["begin"], ev[1]["end"], ev[1]["peak_index"], ev[1]["snr"], ev[1]["boxcar"] = 3, 4, 3, 8, 3
    got, total = _check(ev, dms)  # boxcar 8 at 3: span [4, 12) meets [10, 11)
    assert total == 1 and got[0]["window"] == 4 and got[0]["boxcar_length"] == 8
    ev[1]["boxcar"] = 2  # span [4, 8): apart
    _, total = _check(ev, dms)
    assert total == 2


def test_cluster_representative_ties():
    dms = [5.0, 5.0, 6.0]
    ev = np.zeros(4, EV)
    for i, (trial, b, begin) in enumerate([(2, 0, 50), (1, 1, 50), (1, 0, 51), (1, 0, 49)]):
        ev[i]["trial"], ev[i]["boxcar"], ev[i]["begin"], ev[i]["end"] = trial, b, begin, begin + 3
        ev[i]["peak_index"], ev[i]["snr"] = begin, 9.0
    got, _ = _check(ev, dms)
    assert len(got) == 1 and got[0]["trial"] == 1 and got[0]["boxcar_length"] == 1 and got[0]["peak_index"] == 49


@pytest.mark.parametrize("cap", [0, 1, 7])
def test_cluster_truncation(cap):
    rng = np.random.default_rng(11)
    ev = _random_events(rng, 300, 6, 2, t_max=400)
    dms = np.linspace(0, 10, 6).astype(np.float32)
    _check(ev, dms, cap)


def test_cluster_argument_errors():
    lib = sb.load_library()
    dms = (C.c_float * 2)(1.0, 2.0)
    n = C.c_uint64()
    ev = np.zeros(1, EV)
    ev[0]["end"] = 1
    out = np.zeros(4, sb._dtype_of(sb.Candidate))
    assert lib.srtb_b200_cluster_events(ev.ctypes.data, 1, dms, 2, out.ctypes.data, 4, None) == -1
    assert lib.srtb_b200_cluster_events(None, 1, dms, 2, out.ctypes.data, 4, C.byref(n)) == -1
    assert lib.srtb_b200_cluster_events(ev.ctypes.data, 1, None, 2, out.ctypes.data, 4, C.byref(n)) == -1
    assert lib.srtb_b200_cluster_events(ev.ctypes.data, 1, dms, 0, out.ctypes.data, 4, C.byref(n)) == -1
    assert lib.srtb_b200_cluster_events(ev.ctypes.data, 1, dms, 2, None, 4, C.byref(n)) == -1
    assert lib.srtb_b200_cluster_events(None, 0, dms, 2, None, 0, C.byref(n)) == 0 and n.value == 0
    for field, value in [("trial", 2), ("boxcar", 32), ("end", 0)]:
        bad = ev.copy()
        bad[0][field] = value
        assert lib.srtb_b200_cluster_events(bad.ctypes.data, 1, dms, 2, out.ctypes.data, 4, C.byref(n)) == -1


def test_struct_layouts():
    assert C.sizeof(sb.Event) == 40
    assert [getattr(sb.Event, f).offset for f, _ in sb.Event._fields_] == [0, 8, 16, 24, 28, 32, 36]
    assert C.sizeof(sb.Candidate) == 72
    assert [getattr(sb.Candidate, f).offset for f, _ in sb.Candidate._fields_] == [0, 4, 8, 12, 16, 24, 32, 40, 48,
                                                                                   56, 64, 68]
    assert EV.itemsize == 40 and sb._dtype_of(sb.Candidate).itemsize == 72


def test_runs_oracle_is_strict():
    v = np.array([0, 2, 3, 3, 1, 2, 2, 0, 5], np.float32)
    assert oracle.runs(v, 1.0, 4.0) == [(1, 4, 2, np.float32(1.5)), (5, 7, 5, np.float32(1.0)),
                                        (8, 9, 8, np.float32(2.5))]
    assert oracle.runs(v, 2.0, 0.0) == [(2, 4, 2, 0.0), (8, 9, 8, 0.0)]


def test_executable_rejects_the_key_without_a_dm_search(tmp_path):
    """src/srtb_b200 refuses dm_search_candidates at start-up, from the command line or a .cfg, naming the three keys
    (the check runs before any device is touched)"""
    import subprocess
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    subprocess.run(["make", "-C", str(root / "src")], check=True, capture_output=True)
    exe = str(root / "src" / "srtb_b200")
    cfg = tmp_path / "k.cfg"
    cfg.write_text("dm_search_candidates = 1\n")
    for args in (["--dm_search_candidates", "1"], ["--config_file_name", str(cfg)]):
        r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=60, cwd=tmp_path)
        assert r.returncode == 2, r.stderr[-2000:]
        msg = r.stderr.strip().splitlines()[-1]
        assert "dm_search_candidates" in msg and "dm_list" in msg and "incoherent_dm_list" in msg, msg
