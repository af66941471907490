"""Host checks of rfi_truth.py and of the GPU case lists of test_gpu_rfi_decisions.py. No GPU needed.

rfi_route must name the kernels the library picks for a geometry (the GPU test then checks that each case launched
them), the case lists must reach every route and every (mean route, SK route) pair a shipped configuration runs, the
mask recovery must find an injected s1 mask exactly, the SK window must match the CPU oracle's bit for bit, and the
spikes of the special-bin cases must carry the power they are meant to.
"""
import numpy as np
import pytest

import rfi_truth as rt
from test_chirp_newton import CONFIG1, CONFIG2, CONFIG3, CONFIG4, GPU_CASES

S1_MARGIN = 1e-5        # relative to the float64 limit
SK_MARGIN = 1e-4        # relative to the nearer window edge

# ------------------------------------------------------------------------------------- the GPU case lists
# group A, the route matrix: (name, n, C, f_low, bw, dm, bits); int8 noise, avg_thr 1.5, manual ranges across a
# channel edge, sk_thr from the case's float64 SK
ROUTE_CASES = [c + (-8,) for c in GPU_CASES] + [
    ("post_8192_row8", 1 << 13, 8, 1000.0, 500.0, 56.778, -8),
    ("fixup2_65536_row16", 1 << 16, 32, 1000.0, 500.0, 56.778, -8),
    ("fixup2_131072_bigrow", 1 << 17, 8, 1000.0, 500.0, 56.778, -8),
    ("fixup2_262144_row16", 1 << 18, 64, 1000.0, 500.0, 56.778, -8),
    ("fixup4_2p28_long", 1 << 28, 1 << 11, 1000.0, 500.0, 56.778, -8),
    ("unpacked_int16_row16", 1 << 22, 512, 1000.0, 400.0, 562.05, -16),
]
# group B, the bins the mean kernels treat specially: one geometry per mean route of the split (n, C)
SPIKE_GEOMS = {"post": (1 << 20, 256), "fixup2": (1 << 17, 16), "fixup3": (1 << 22, 256), "fixup4": (1 << 28, 1 << 11)}
# group C, streams of unequal power: (name, n per stream, C, format name, f_low, bw, dm)
STREAM_CASES = [
    ("naocpsr_snap1_bigrow", 1 << 22, 256, "naocpsr_snap1", 1000.0, 64.0, 500.0),
    ("interleaved_2_row16", 1 << 22, 512, "interleaved_samples_2", 1000.0, 400.0, 562.05),
    ("gznupsr_a1_long", 1 << 22, 64, "gznupsr_a1", 1000.0, 64.0, 100.0),
    ("config3_snap1_sweep_order", 1 << 26, 1 << 11, "naocpsr_snap1", 1000.0, 400.0, 562.05),
]
STREAM_FORMATS = {"naocpsr_snap1": rt.NAOCPSR_SNAP1, "interleaved_samples_2": rt.INTERLEAVED_2,
                  "gznupsr_a1": rt.GZNUPSR_A1_2}
# group D, manual ranges on the linear layout: (name, n, C, f_low, bw, dm)
RANGE_CASES = [
    ("ranges_row16", 1 << 20, 512, 1000.0, 500.0, 56.778),
    ("ranges_bigrow_inverted", 1 << 22, 256, 1437.0, -64.0, -478.80),
    ("ranges_long", 1 << 22, 64, 1000.0, 64.0, 100.0),
    ("ranges_unfused", 1 << 20, 4096, 1000.0, 500.0, 56.778),
]

# (n, C, bits, format, path) of the shipped configurations (bench.py WORKLOADS; config5 is config3's R2C on one stream)
SHIPPED = {"config1": (CONFIG1[0], CONFIG1[1], 2, rt.SIMPLE, "block"),
           "config2": (CONFIG2[0], CONFIG2[1], -8, rt.SIMPLE, "block"),
           "config3": (CONFIG3[0], CONFIG3[1], -8, rt.NAOCPSR_SNAP1, "block"),
           "config4": (CONFIG4[0][0], CONFIG4[0][1], -8, rt.SIMPLE, "sweep"),
           "config5": (1 << 26, 1 << 11, -8, rt.SIMPLE, "block")}


def route_case_routes():
    """rfi_route of every group A case on both paths, and of every group C case on both paths"""
    out = {}
    for name, n, C, *_, bits in ROUTE_CASES:
        for path in ("block", "sweep"):
            out[(name, path)] = rt.rfi_route(n, C, bits, rt.SIMPLE, path)
    for name, n, C, fmt, *_ in STREAM_CASES:
        for path in ("block", "sweep"):
            out[(name, path)] = rt.rfi_route(n, C, -8, STREAM_FORMATS[fmt], path)
    return out


EXPECTED_MEAN_ROUTES = {(r, k) for r in ("fixup2", "fixup3", "fixup4") for k in ("raw",)} | {
    ("post", "unpacked"), ("fixup3", "unpacked"), ("rows_split", "raw")}
EXPECTED_SK_PAIRS = {(("fixup4", "raw"), "long"), (("fixup3", "raw"), "row16"), (("rows_split", "raw"), "bigrow"),
                     (("fixup3", "raw"), "long")}


def test_gpu_cases_reach_every_route():
    routes = set(route_case_routes().values())
    assert {r[0] for r in routes} == EXPECTED_MEAN_ROUTES
    assert {r[1] for r in routes} == {"row16", "bigrow", "long", "unfused"}
    assert {r[2] for r in routes} == set(rt.TAIL_ROUTES)
    assert {m[0] for m, *_ in routes} == set(rt.MEAN_ROUTES)
    # the pairs the shipped configurations run
    shipped = {(r[0], r[2]) for r in (rt.rfi_route(*g) for g in SHIPPED.values())}
    assert shipped == EXPECTED_SK_PAIRS
    assert shipped <= {(r[0], r[2]) for r in routes}
    # every mean route of the split has a spike geometry
    assert {rt.rfi_route(n, C, -8, rt.SIMPLE, "block")[0][0] for n, C in SPIKE_GEOMS.values()} == set(SPIKE_GEOMS)
    # every linear-layout s1 route has a manual-range case, and one runs on an inverted band
    assert {rt.rfi_route(c[1], c[2], -8, rt.SIMPLE, "block")[1] for c in RANGE_CASES} == {"row16", "bigrow", "long",
                                                                                           "unfused"}
    assert any(c[4] < 0 for c in RANGE_CASES)


@pytest.mark.parametrize("geom,expect", [
    ((1 << 13, 8, -8, rt.SIMPLE, "block"), (("post", "unpacked"), "unfused", "row8_512")),
    ((1 << 14, 8, -8, rt.SIMPLE, "block"), (("fixup2", "raw"), "row16", "row16")),
    ((1 << 18, 64, -8, rt.SIMPLE, "sweep"), (("fixup2", "raw"), "row16", "row16")),
    ((1 << 19, 32, -8, rt.SIMPLE, "block"), (("post", "unpacked"), "bigrow", "bigrow")),
    ((1 << 21, 2, -8, rt.SIMPLE, "block"), (("post", "unpacked"), "unfused", "unfused")),
    ((1 << 22, 512, -16, rt.SIMPLE, "block"), (("fixup3", "unpacked"), "row16", "row16")),
    ((1 << 22, 512, 32, rt.SIMPLE, "sweep"), (("fixup3", "unpacked"), "row16", "row16")),
    ((1 << 22, 64, 8, rt.NAOCPSR_SNAP1, "block"), (("fixup3", "unpacked"), "long", "long")),   # snap1 is int8 only
    ((1 << 23, 64, 4, rt.SIMPLE, "block"), (("fixup3", "raw"), "long", "long")),
    ((1 << 26, 1 << 11, 4, rt.SIMPLE, "block"), (("fixup3", "unpacked"), "bigrow", "bigrow")),  # 2^9: no packed variant
    ((CONFIG1[0], CONFIG1[1], 2, rt.SIMPLE, "block"), (("fixup4", "raw"), "long", "long")),
    ((CONFIG2[0], CONFIG2[1], -8, rt.SIMPLE, "block"), (("fixup3", "raw"), "row16", "row16")),
    ((CONFIG2[0], CONFIG2[1], -8, rt.SIMPLE, "sweep"), (("fixup3", "raw"), "row16", "row16")),
    ((CONFIG3[0], CONFIG3[1], -8, rt.NAOCPSR_SNAP1, "block"), (("rows_split", "raw"), "bigrow", "bigrow")),
    ((CONFIG3[0], CONFIG3[1], -8, rt.NAOCPSR_SNAP1, "sweep"), (("fixup3", "raw"), "bigrow", "bigrow")),
    ((CONFIG4[0][0], CONFIG4[0][1], -8, rt.SIMPLE, "block"), (("fixup3", "raw"), "long", "long")),
    ((CONFIG4[0][0], CONFIG4[0][1], -8, rt.SIMPLE, "sweep"), (("fixup3", "raw"), "long", "long")),
    ((1 << 28, 1 << 11, -8, rt.SIMPLE, "sweep"), (("fixup4", "raw"), "long", "long")),
    ((1 << 26, 1 << 11, 2, rt.SIMPLE, "block"), (("fixup3", "unpacked"), "bigrow", "bigrow")),  # sweep order: 8-bit
    ((1 << 26, 1 << 11, -8, rt.INTERLEAVED_2, "block"), (("rows_split", "raw"), "bigrow", "bigrow")),
    ((1 << 20, 4096, -8, rt.SIMPLE, "block"), (("post", "unpacked"), "unfused", "unfused")),
])
def test_route_selection(geom, expect):
    assert rt.rfi_route(*geom) == expect


def test_window_forces_the_unpack_kernel():
    assert rt.rfi_route(1 << 24, 2048, -8, rt.SIMPLE, "block", window=1)[0] == ("fixup3", "unpacked")


# ------------------------------------------------------------------------------------------------ the truth
def _chain(X, mask, coef, C, chirp):
    """float64 dynamic spectrum [C][L] of spectrum X with the bins of `mask` zapped"""
    Z = np.where(mask, 0, X * coef) * chirp
    return np.fft.ifft(Z.reshape(C, -1), axis=1) * (Z.size // C)


def test_recover_s1_mask_finds_an_injected_mask():
    """a float64 chain with a known mask, rounded to complex64 and perturbed by 1e-6 relative noise: the recovered
    mask equals the injected one on every bin that is not ambiguous"""
    rng = np.random.default_rng(5)
    n, C = 1 << 16, 16
    bb = rt.noise_int8(n, 6)
    X = np.fft.rfft(bb.astype(np.float64))[:n // 2]
    mask, limit, pw = rt.s1_truth(X, 1.5, [(1000, 1100), (4095, 4096)])
    assert 0.15 < mask.mean() < 0.3
    coef = 1.0 / np.sqrt((n // 2) ** 2 / C)
    chirp = np.exp(2j * np.pi * rng.random(n // 2))
    y = _chain(X, mask, coef, C, chirp)
    y = y + 1e-6 * np.sqrt(np.mean(np.abs(y) ** 2)) * (rng.standard_normal(y.shape) + 1j * rng.standard_normal(y.shape))
    got, amb = rt.recover_s1_mask(y.astype(np.complex64), X.reshape(C, -1), coef, pw.mean())
    amb = amb.reshape(-1)
    print(f"recovered {int(got.sum())} zapped bins of {got.size}, {int(amb.sum())} ambiguous")
    assert amb.sum() < 1e-4 * amb.size
    assert np.array_equal(got.reshape(-1)[~amb], mask[~amb])
    # one flipped bin of the chain is found, and reported as a flip far from the edge
    flipped = mask.copy()
    k = int(np.nonzero(~mask & (pw > 0.5 * limit))[0][0])
    flipped[k] = True
    got2, _ = rt.recover_s1_mask(_chain(X, flipped, coef, C, chirp).astype(np.complex64), X.reshape(C, -1), coef,
                                 pw.mean())
    d = rt.compare_decisions(got2.reshape(-1)[~amb], pw[~amb], limit, S1_MARGIN, truth=mask[~amb])
    assert d.flips == 1 and d.worst > 0.1


def test_compare_decisions_counts_flips_and_informative_band():
    stat = np.array([1.0, 1.5 * (1 + 5e-6), 1.5 * (1 - 5e-4), 1.5 * (1 + 0.5), np.nan])
    got = np.array([False, False, False, True, False])
    d = rt.compare_decisions(got, stat, 1.5, S1_MARGIN)
    assert (d.total, d.flips, d.informative) == (5, 1, 1) and d.worst == pytest.approx(5e-6, rel=1e-6)
    lo, hi = rt.sk_window(1.05, 4096)
    sk = np.array([lo * (1 - 2e-3), hi * (1 + 5e-5), 2.0, np.nan])
    d = rt.compare_decisions(np.array([True, False, False, False]), sk, (lo, hi), SK_MARGIN)
    assert (d.flips, d.informative) == (1, 1) and d.worst < SK_MARGIN


def test_sk_truth_of_rows():
    rng = np.random.default_rng(2)
    y = (rng.standard_normal((64, 4096)) + 1j * rng.standard_normal((64, 4096))) / np.sqrt(2)
    sk = rt.sk_truth(y)
    assert abs(sk.mean() - 2) < 0.02
    y[3] = 0
    y[5, 1:] = 0
    sk = rt.sk_truth(y)
    assert np.isnan(sk[3]) and sk[5] == pytest.approx(4096)


@pytest.mark.parametrize("thr", [0.5, 0.97, 1.0, 1.05, 1.3, 1.95, 2.0, 2.5, 3.0])
@pytest.mark.parametrize("M", [1, 2, 511, 512, 4096, 16384, 1 << 18, (1 << 18) + 3])
def test_sk_window_matches_the_oracle(oracle, thr, M):
    """bit for bit, the swap branch (thr < 1) and a negative lower edge (thr > 2) included"""
    lo, hi = rt.sk_window(thr, M)
    assert (lo, hi) == oracle.sk_thresholds(M, thr)
    assert lo <= hi
    if thr > 2 and M > 1:     # 2 - thr < 0: the lower edge lies below 1, under any SK (SK >= 1 by Cauchy-Schwarz)
        assert lo < 1


def test_sk_window_swap_branch():
    """thr < 1 gives the window of 2 - thr, up to the float32 rounding of 2 - thr"""
    assert rt.sk_window(0.97, 4096) == rt.sk_window(float(np.float32(2) - np.float32(0.97)), 4096)


@pytest.mark.parametrize("route", ["post", "fixup2", "fixup3"])
@pytest.mark.parametrize("kind", rt.SPIKES)
def test_spikes_carry_their_power(route, kind):
    """each spike of group B puts 1 - 5 % of the block's power into its bin, and the bins are the intended ones
    (column 0 of the fused split or not). The 2^28 geometry of fixup4 is checked on the device by the GPU test."""
    n, _ = SPIKE_GEOMS[route]
    samples = rt.with_spike(rt.noise_int8(n, 40), kind)
    frac = rt.spike_fraction(samples, kind)
    base = rt.spike_fraction(rt.noise_int8(n, 40), kind)
    print(f"{route} {kind}: bin {rt.spike_bin(n, kind)} holds {frac:.4f} of the power ({base:.1e} without the spike)")
    assert 0.01 <= frac <= 0.05
    assert base < 1e-4
    k, l1 = rt.spike_bin(n, kind), rt.first_sweep(n)
    if kind == "col0":
        assert k % (1 << l1) == 0 and 0 < k < n // 4
    if kind == "generic":
        assert k % (1 << l1) != 0


def test_spike_bins_at_the_fixup4_geometry():
    n = SPIKE_GEOMS["fixup4"][0]
    l1 = rt.first_sweep(n)
    assert l1 == 7
    assert rt.spike_bin(n, "col0") % (1 << l1) == 0 and rt.spike_bin(n, "generic") % (1 << l1) != 0
    assert rt.spike_bin(n, "half") == n // 4 and rt.spike_bin(n, "nyquist") == n // 2
