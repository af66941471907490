"""Restatements of the single-pulse event list and its candidates (include/srtb_b200.h, srtb_b200_event and
srtb_b200_cluster_events), for the tests.

runs(v, thr, var): every maximal run of v > thr, exact on the given float32 values.
cluster(events, dms): friends of friends by direct pairwise comparison and a plain union-find (no sweep), so it shares
no logic with the library's O(n log n) sweep.
"""
from __future__ import annotations

import numpy as np


def runs(v, thr, var):
    """[(begin, end, peak_index, snr)] of the maximal runs of v[j] > thr (float32 compare), in order. snr is the run's
    largest value over sqrt(var) in float32 (0 when var is 0); peak_index its smallest index."""
    v = np.asarray(v, np.float32)
    above = v > np.float32(thr)
    if not above.any():
        return []
    d = np.diff(np.concatenate(([0], above.astype(np.int8), [0])))
    begins = np.flatnonzero(d == 1)
    ends = np.flatnonzero(d == -1)
    out = []
    var32 = np.float32(var)
    for b, e in zip(begins, ends):
        seg = v[b:e]
        k = int(np.argmax(seg))  # first index of the maximum
        m = seg[k]
        snr = np.float32(m / np.sqrt(var32)) if var32 > 0 else np.float32(0)
        out.append((int(b), int(e), int(b) + k, snr))
    return out


def span(e):
    o = 1 if int(e["boxcar"]) else 0
    return int(e["begin"]) + o, int(e["end"]) - 1 + o + (1 << int(e["boxcar"]))


def cluster(events, dms):
    """list of candidate dicts in output order (the fields of srtb_b200_candidate)"""
    n = len(events)
    order = sorted(range(len(dms)), key=lambda d: np.float32(dms[d]))  # stable
    rank = np.empty(len(dms), np.int64)
    rank[order] = np.arange(len(dms))
    lo = np.array([span(e)[0] for e in events], np.int64)
    hi = np.array([span(e)[1] for e in events], np.int64)
    st = np.array([int(e["stream"]) for e in events], np.int64)
    rk = np.array([rank[int(e["trial"])] for e in events], np.int64)
    parent = list(range(n))

    def find(i):
        while parent[i] != i:
            i = parent[i]
        return i

    for i in range(n):
        f = (st == st[i]) & (np.abs(rk - rk[i]) <= 1) & (lo < hi[i]) & (lo[i] < hi)
        for j in np.flatnonzero(f[:i]):
            a, b = find(i), find(int(j))
            if a != b:
                parent[max(a, b)] = min(a, b)
    groups = {}
    for i in range(n):
        groups.setdefault(find(i), []).append(i)
    cands = []
    for members in groups.values():
        def key(i):
            e = events[i]
            return (-float(e["snr"]), int(e["trial"]), int(e["boxcar"]), int(e["begin"]))
        r = min(members, key=key)
        e = events[r]
        o = 1 if int(e["boxcar"]) else 0
        mdms = [np.float32(dms[int(events[i]["trial"])]) for i in members]
        cands.append(dict(snr=np.float32(e["snr"]), dm=np.float32(dms[int(e["trial"])]), dm_low=min(mdms),
                          dm_high=max(mdms), boxcar_length=1 << int(e["boxcar"]), peak_index=int(e["peak_index"]),
                          window=int(e["peak_index"]) + o, members=len(members),
                          span_begin=int(lo[members].min()), span_end=int(hi[members].max()), trial=int(e["trial"]),
                          stream=int(e["stream"]), _begin=int(e["begin"])))
    cands.sort(key=lambda c: (c["stream"], c["span_begin"], c["trial"], c["boxcar_length"], c["_begin"]))
    for c in cands:
        del c["_begin"]
    return cands
