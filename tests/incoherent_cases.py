"""The trial lists and geometries the incoherent DM search's GPU tests run at (tests/test_gpu_incoherent_geometry.py),
each named for the grouping structure it is meant to reach. tests/test_incoherent_groups.py checks on the CPU, with the
grouping restatement of tests/incoherent_grouping.py, that every case reaches it.

All cases but the long-series ones run at config #3's stream shape: C = 2048 channels, 1 GHz sampling, f_low = 1000 MHz,
|bandwidth| = 500 MHz, dm = 100. One DM unit then moves the band edge by about 562 samples with an upright band
(f_ref = 1500 MHz) and by about 3000 with an inverted one (f_ref = 500 MHz)."""
from __future__ import annotations

import numpy as np

import incoherent_oracle as io

C, L, SR, DM = 2048, 16384, 1e9, 100.0
BANDS = {"upright": (1000.0, 500.0), "inverted": (1000.0, -500.0)}


def _f32(v) -> float:
    return float(np.float32(v))


def _edge_spread(band: str, a: float, b: float) -> int:
    """the largest |s[b][c] - s[a][c]| over the channels"""
    s, _, _ = io.shifts(C, *BANDS[band], SR, DM, [a, b])
    return int(np.abs(s[1] - s[0]).max())


def dm_at_spread(band: str, a: float, target: int) -> float:
    """the smallest float32 DM above a whose shifts differ from a's by `target` on some channel (bisection over the
    float32 bit patterns, which order positive floats)"""
    lo = int(np.float32(a).view(np.int32))
    hi = int(np.float32(a + 4.0 * target / 500.0).view(np.int32))
    assert _edge_spread(band, a, float(np.int32(hi).view(np.float32))) >= target
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _edge_spread(band, a, float(np.int32(mid).view(np.float32))) >= target:
            hi = mid
        else:
            lo = mid
    b = float(np.int32(hi).view(np.float32))
    assert _edge_spread(band, a, b) == target, (band, a, target)
    return b


def _upright_dms():
    """a dense run cut by count (80 trials 0.01 apart), a sparse run cut by spread (0.1 apart) and three trials 3.3 DM
    apart, each a group of its own"""
    dense = [DM - 1.0 + 0.01 * i for i in range(80)]
    sparse = [DM - 0.2 + 0.1 * i for i in range(65)]
    single = [DM + 9.5, DM + 12.8, DM + 16.1]
    return [_f32(d) for d in dense + sparse + single]


def _inverted_dms():
    """under one DM unit: a dense run cut by count (100 trials 0.002 apart), then a sparse one cut by spread (0.02
    apart, 60 samples at the edge)"""
    dense = [DM - 0.2 + 0.002 * i for i in range(100)]
    sparse = [DM + 0.02 * i for i in range(40)]
    return [_f32(d) for d in dense + sparse]


def _spread_1792_dms():
    """group 0 runs from DM to the trial 1792 samples away at the edge; the next trial would make it 1793"""
    b = dm_at_spread("upright", DM, 1792)
    b1 = dm_at_spread("upright", DM, 1793)
    mid = [_f32(DM + 0.5 * i) for i in range(1, 6)]
    return [_f32(DM)] + mid + [b, b1, _f32(b1 + 0.5), _f32(b1 + 1.0)]


def _spread_dms(target: int):
    """one group whose largest spread is `target`"""
    b = dm_at_spread("upright", DM, target)
    return [_f32(DM)] + [_f32(DM + 0.4 * i) for i in range(1, 6)] + [b]


def _tail_dms():
    """40 trials over +-0.3 DM of an inverted band: two groups, cut by spread"""
    return [_f32(DM + d) for d in np.linspace(-0.3, 0.3, 40)]


def span(band: str, dms) -> int:
    _, sp, sm = io.shifts(C, *BANDS[band], SR, DM, dms)
    return sp + sm


def _case(band, dms, time_count=L, reserved=None, T=None, residue=None):
    """reserved (the detector's tail) or T, or the T residue modulo 256 with time_count = span + T"""
    sp = span(band, dms)
    if T is not None:
        time_count, reserved = sp + T + (reserved or 0), reserved or 0
    elif residue is not None:  # the largest T <= L - span with that residue, reserved = 0
        T = L - sp - ((L - sp - residue) % 256)
        time_count, reserved = sp + T, 0
    return {"band": band, "dms": list(dms), "time_count": time_count, "reserved": reserved}


def cases() -> dict:
    up, inv = _upright_dms(), _inverted_dms()
    rng = np.random.default_rng(5)
    shuffled = list(up)
    rng.shuffle(shuffled)
    dup = up[:40] + up[30:60] + up[40:]  # trials 30..59 twice: ties the stable sort keeps in list order
    rng.shuffle(dup)
    up_sp = span("upright", up)
    return {
        # T = L - reserved - span, reserved chosen so that T = 0 mod 256 (upright) / an odd residue (inverted)
        "upright": _case("upright", up, reserved=(L - up_sp) % 256),
        "inverted": _case("inverted", inv, reserved=100),
        "spread_1792": _case("upright", _spread_1792_dms(), reserved=0),
        "smem_1472": _case("upright", _spread_dms(1472), reserved=0),
        "smem_1473": _case("upright", _spread_dms(1473), reserved=0),
        "shuffled": _case("upright", shuffled, reserved=(L - up_sp) % 256),
        "reversed": _case("upright", up[::-1], reserved=(L - up_sp) % 256),
        "duplicates": _case("upright", dup, reserved=(L - up_sp) % 256),
        "tail_1": _case("inverted", _tail_dms(), residue=1),
        "tail_255": _case("inverted", _tail_dms(), residue=255),
        "short": _case("inverted", _tail_dms(), T=200, reserved=3),
    }


# series longer than gridDim.y's 65535 tiles of 256: C = 2, three trials, 1 MHz sampling (shifts of a few hundred)
LONG_C, LONG_SR, LONG_BAND = 2, 1e6, (1000.0, 500.0)
LONG_DMS = [_f32(DM - 0.3), _f32(DM), _f32(DM + 0.4)]
LONG_T = {"65535_tiles": 65535 * 256, "65535_tiles_plus_1": 65535 * 256 + 1, "2^24+2^17": (1 << 24) + (1 << 17)}


def long_span() -> int:
    _, sp, sm = io.shifts(LONG_C, *LONG_BAND, LONG_SR, DM, LONG_DMS)
    return sp + sm
