"""Restatement of the incoherent DM search's trial grouping (incoherent_grouping in csrc/srtb_b200.cu), for the tests.

The dedispersion kernel forms up to INC_GROUP trials per CTA from one staged span per channel, so the host sorts the
trials by DM and cuts the sorted list into groups whose shift spread fits the staging buffer. The shifts s [n_dm][C] are
tests/incoherent_oracle.py's."""
from __future__ import annotations

import numpy as np

INC_TILE, INC_GROUP, INC_SPREAD_MAX, INC_STAGES = 256, 64, 1792, 3  # the dedispersion kernel's constants


def groups(s: np.ndarray, dms):
    """the float32 DMs stably sorted, then cut greedily into groups of at most INC_GROUP trials whose spread
    max s - min s over the group is at most INC_SPREAD_MAX on every channel (a trial that would break either limit
    starts the next group). Returns (order [n_dm] trial of each sorted slot, [(first slot, count)] per group,
    gmin [groups][C], gmax [groups][C] of s over each group, the largest spread)."""
    order = np.argsort(np.asarray(dms, np.float32), kind="stable")
    out, gmins, gmaxs = [], [], []
    first = 0
    while first < len(order):
        gmin = s[order[first]].copy()
        gmax = gmin.copy()
        count = 1
        while first + count < len(order) and count < INC_GROUP:
            row = s[order[first + count]]
            nmin, nmax = np.minimum(gmin, row), np.maximum(gmax, row)
            if np.any(nmax - nmin > INC_SPREAD_MAX):
                break
            gmin, gmax = nmin, nmax
            count += 1
        out.append((first, count))
        gmins.append(gmin)
        gmaxs.append(gmax)
        first += count
    gmin, gmax = np.array(gmins), np.array(gmaxs)
    return order, out, gmin, gmax, int((gmax - gmin).max())


def smem_bytes(spread: int) -> int:
    """incoherent_smem_bytes: the kernel's dynamic shared memory for a largest group spread `spread`"""
    return (INC_TILE + spread) * (INC_STAGES * 8 + 4) + INC_STAGES * INC_GROUP * 4
