"""Host mirror of how the library picks a chirp route and reciprocal variant, and a float64 emulation of the Newton
reciprocal chains the on-the-fly chirp kernels walk. No GPU needed.

The coherent-dedispersion phase of bin i is k = ddm / f * ((f - f_c) / f_c)^2 cycles, f = f_min + df i. Where the
phase is evaluated on the fly (the DM sweep, and long rows on both entry points), 1/f comes from one correctly rounded
reciprocal per thread and Newton steps r' = r + r (1 - f r) from a neighbouring bin. After n steps the relative error
of r is about delta^(2^n), delta being the neighbours' relative distance; the host picks n so that
|k| delta^(2^n) < 1e-9 cycles (DESIGN.md, the whole-row kernel). The tests below restate that selection and walk the
chains with exactly emulated fused multiply-adds, so a dropped step, a wrong stride or a rule that picks too few steps
shows up as a phase error here, before any GPU run.
"""
import numpy as np
import pytest

D_E6 = 4.148808e3 * 1e6          # dispersion constant (MHz^2 pc^-1 cm^3 s) times 1e6: k in cycles for f in MHz
EPS = 2.0 ** -52
PHASE_BOUND = 1e-9               # cycles: the Newton truncation error the selection promises
ROUNDING_ULPS = 4                # allowance in ulp of |k| for the roundings of the chain itself
DROPPED_STEP_RMS = 2e-6          # cycles: an RMS phase error of 2 pi * 2e-6 rad already exceeds the 1e-5 rel-L2 bound

ROW16 = (1 << 10, 1 << 11, 1 << 12)          # sixteen-point row kernel with the chirp on load
BIGROW = (1 << 13, 1 << 14)                  # whole-row kernel
LONG = tuple(1 << q for q in range(15, 19))  # column sweep with the chirp on load + transposing last sweep


class ChirpParams:
    """row geometry and the doubles of row_chirp_params, with the float32 roundings block_params_for applies
    (f_min, f_c = f_min + bw and df = bw / Nc are float32; the DM crosses as float32)"""

    def __init__(self, n, C, f_low, bw, dm):
        self.nc = n // 2
        self.C = min(C, self.nc)
        self.L = self.nc // self.C
        f_min = np.float32(f_low)
        bw32 = np.float32(bw)
        self.f_min = float(f_min)
        self.df = float(np.float32(bw32 / np.float32(self.nc)))
        self.f_c = float(np.float32(f_min + bw32))
        self.inv_fc = 1.0 / self.f_c
        self.ddm = D_E6 * float(np.float32(dm))
        # fa, q, kmax: the bounds both selection rules start from (kmax >= |k| over the band)
        self.fa = min(abs(self.f_min), abs(self.f_c))
        q = (self.f_c - self.f_min) * self.inv_fc
        self.kmax = max(1.0, abs(self.ddm) / self.fa * q * q)


def _steps(d2, kmax):
    """Newton steps for neighbours a relative distance sqrt(d2) apart: 1 when one step is good to an ulp, 2 when the
    fourth power keeps the phase error below 1e-9 cycles, 0 = the exact reciprocal of every bin"""
    return 1 if d2 <= EPS else (2 if d2 * d2 * kmax < PHASE_BOUND else 0)


def bigrow_steps(p):
    """(far, near) steps of the whole-row kernel: far = B1 = L/16 bins along a butterfly's inputs, near = the adjacent
    bin (srtb_b200.cu, watfft_sk_detect_fused, lines 1558-1573)"""
    far = (p.L // 16) * abs(p.df) / p.fa
    near = abs(p.df) / p.fa
    return _steps(far * far, p.kmax), _steps(near * near, p.kmax)


def long_geometry(L):
    """first (column) and last sweep lengths of the long-row plan (srtb_b200.cu, watfft_long_fused)"""
    q = L.bit_length() - 1
    l1 = (q + 1) // 2
    return 1 << l1, 1 << (q - l1)


def long_steps(p):
    """cp.newton of the long-row column sweep: points U B = (L1 / 16) L2 bins apart (srtb_b200.cu, lines 1622-1628)"""
    L1, L2 = long_geometry(p.L)
    d = (L1 // 16) * L2 * abs(p.df) / p.fa
    return _steps(d * d, p.kmax)


def chirp_variant(n, C, f_low, bw, dm, path):
    """(route, variant) the library runs for stream_tail at this geometry; path = "block" (process_block) or "sweep"
    (process_block_dm_sweep). Routes: "row16" (variant "table" or "fly": chirp_factor on the fly), "bigrow" (the
    kernel's CHIRP: 5 = phase table, 1 / 3 / 4 = Newton steps, 2 = exact reciprocal), "long" (cp.newton: 0 = exact,
    1 or 2 steps), "unfused" (dedisperse_kernel before a plain waterfall; variant None). Buffers are taken to be
    16-byte aligned and TMA descriptors available, as they are for the library's own buffers on an H100."""
    assert path in ("block", "sweep")
    p = ChirpParams(n, C, f_low, bw, dm)
    table = path == "block" and p.nc * 4 <= (4 << 30)   # get_chirp_table keeps no table above 4 GiB
    if p.L in ROW16:
        return "row16", "table" if table else "fly"
    if p.L in BIGROW:
        if table:
            return "bigrow", 5
        far, near = bigrow_steps(p)
        if far == 0 or near == 0:
            return "bigrow", 2
        return "bigrow", 1 if far == 1 else (3 if near == 1 else 4)
    if p.L in LONG:
        return "long", long_steps(p)
    return "unfused", None


# ---------------------------------------------------------------------------------------------- exact fp64 emulation
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a                  # 2^27 + 1 (Veltkamp)
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma(a, b, c):
    """a * b + c rounded once (float64 arrays). The product is split exactly; the three-term sum is rounded once except
    when it lies within 2^-106 (relative) of a rounding boundary, which the bounds below never depend on."""
    p, e = _two_prod(np.asarray(a, np.float64), np.asarray(b, np.float64))
    s, t = _two_sum(p, np.asarray(c, np.float64))
    return s + (t + e)


def newton(r, f, steps):
    for _ in range(steps):
        r = fma(r, fma(-f, r, 1.0), r)
    return r


def _refine(r, f, steps):
    return 1.0 / f if steps == 0 else newton(r, f, steps)     # 0: __drcp_rn, the correctly rounded reciprocal


def bigrow_reciprocals(p, row, far, near):
    """(f, 1/f) of every bin of channel row `row`, bin order, as fft_bigrow_kernel's stage 0 walks them: thread tid takes
    bins j = 2 tid and j + 1 of each of the sixteen chunks; 1/f of bin j + i B1 comes from bin j + (i - 1) B1 by `far`
    steps, that of bin j + i B1 + 1 from bin j + i B1 by `near` steps (0 = exact)"""
    L, B1 = p.L, p.L // 16
    idx = float(row * L) + 2.0 * np.arange(L // 32)
    f = np.empty((16, 2, L // 32))
    r = np.empty_like(f)
    fa = fma(p.df, idx, p.f_min)
    ra = 1.0 / fa
    for i in range(16):
        if i > 0:
            idx = idx + B1
            fa = fma(p.df, idx, p.f_min)
            ra = _refine(ra, fa, far)
        fb = fma(p.df, idx + 1.0, p.f_min)
        f[i, 0], r[i, 0] = fa, ra
        f[i, 1], r[i, 1] = fb, _refine(ra, fb, near)
    # [i][pair][tid] -> bin i B1 + 2 tid + pair
    return f.transpose(0, 2, 1).reshape(L), r.transpose(0, 2, 1).reshape(L)


def long_reciprocals(p, row, steps):
    """(f, 1/f) of every bin of channel row `row` as fft_col16_tma_kernel<..., CH> walks them: the thread of column
    b0 + t, slot u (u < U = L1 / 16) starts at bin row L + u L2 + b0 + t and steps U L2 = L / 16 bins sixteen times"""
    L1, L2 = long_geometry(p.L)
    step = (L1 // 16) * L2
    idx = float(row * p.L) + np.arange(step, dtype=np.float64)
    f = np.empty((16, step))
    r = np.empty_like(f)
    cur_f = fma(p.df, idx, p.f_min)
    cur_r = 1.0 / cur_f
    for e in range(16):
        if e > 0:
            idx = idx + step
            cur_f = fma(p.df, idx, p.f_min)
            cur_r = _refine(cur_r, cur_f, steps)
        f[e], r[e] = cur_f, cur_r
    return f.reshape(p.L), r.reshape(p.L)


def phase_error(p, f, r):
    """(|k(r) - k(1/f)| in cycles, |k|) for each bin: the chirp phase's error from an inexact reciprocal"""
    q = (f - p.f_c) * p.inv_fc
    g = np.abs(p.ddm) * q * q
    return g * np.abs(r - 1.0 / f), g / np.abs(f)


def chain_reciprocals(p, route, variant, row, drop_far=0):
    """reciprocals of one row for an on-the-fly (route, variant); drop_far removes steps from the far chain (the
    whole-row kernel's refine_far, the long-row CH chain)"""
    if route == "bigrow":
        far, near = {1: (1, 1), 2: (0, 0), 3: (2, 1), 4: (2, 2)}[variant]
        return bigrow_reciprocals(p, row, max(far - drop_far, 0) if far else 0, near)
    assert route == "long"
    return long_reciprocals(p, row, max(variant - drop_far, 0) if variant else 0)


def sampled_rows(C, count=3):
    return sorted(set(np.linspace(0, C - 1, count).round().astype(int).tolist()))


# ------------------------------------------------------------------------------------------------- the configurations
# BASELINE.json configs (bench.py WORKLOADS): (n, C, f_low, bw, dm)
CONFIG1 = (1 << 30, 1 << 11, 1437.0, -64.0, -478.80)
CONFIG2 = (1 << 24, 1 << 11, 1000.0, 500.0, 56.778)
CONFIG3 = (1 << 26, 1 << 11, 1000.0, 400.0, 562.05)
CONFIG4_DMS = [0.0, 56.78] + [50.0 * i for i in range(2, 21)]
CONFIG4 = [(1 << 27, 1 << 11, 1000.0, 500.0, dm) for dm in CONFIG4_DMS]

# the GPU route tests (test_gpu_chirp_routes.py): (name, n, C, f_low, bw, dm); every block at most 2^24 samples
GPU_CASES = [
    ("row16_1024", 1 << 20, 512, 1000.0, 500.0, 56.778),
    ("row16_2048_inverted", 1 << 20, 256, 1437.0, -64.0, -478.80),
    ("row16_4096", 1 << 22, 512, 1000.0, 400.0, 562.05),
    ("bigrow_exact_8192", 1 << 20, 64, 1000.0, 500.0, 56.778),
    ("bigrow_v1_8192", 1 << 24, 1024, 1000.0, 0.2, 500.0),
    ("bigrow_v3_16384", 1 << 24, 512, 1000.0, 64.0, 500.0),
    ("bigrow_v4_8192_inverted", 1 << 22, 256, 1437.0, -64.0, -478.80),
    ("long_n2_32768", 1 << 22, 64, 1000.0, 64.0, 100.0),
    ("long_n1_32768", 1 << 24, 256, 1000.0, 0.05, 3000.0),
    ("long_n2_65536", 1 << 22, 32, 1000.0, 64.0, 100.0),
    ("long_n0_131072_inverted", 1 << 22, 16, 1437.0, -64.0, -478.80),
    ("long_n2_131072", 1 << 23, 32, 1000.0, 64.0, 100.0),
    ("long_n2_262144", 1 << 24, 32, 1000.0, 64.0, 100.0),
    ("unfused_512", 1 << 20, 1024, 1000.0, 500.0, 56.778),
    ("unfused_524288", 1 << 22, 4, 1000.0, 500.0, 56.778),
]

EXPECTED_PAIRS = {("row16", "table"), ("row16", "fly"), ("bigrow", 5), ("bigrow", 1), ("bigrow", 2), ("bigrow", 3),
                  ("bigrow", 4), ("long", 0), ("long", 1), ("long", 2), ("unfused", None)}


def gpu_case_pairs():
    return {chirp_variant(*c[1:], path) for c in GPU_CASES for path in ("block", "sweep")}


@pytest.mark.parametrize("geom,path,expect", [
    ((1 << 20, 64, 1000.0, 500.0, 56.778), "sweep", ("bigrow", 2)),
    ((1 << 20, 64, 1000.0, 500.0, 0.02), "sweep", ("bigrow", 4)),
    ((1 << 24, 512, 1000.0, 64.0, 500.0), "sweep", ("bigrow", 3)),
    ((1 << 22, 256, 1437.0, -64.0, -478.80), "sweep", ("bigrow", 4)),
    ((1 << 24, 1024, 1000.0, 0.2, 500.0), "sweep", ("bigrow", 1)),
    ((1 << 24, 512, 1000.0, 64.0, 500.0), "block", ("bigrow", 5)),
    ((1 << 22, 64, 1000.0, 64.0, 100.0), "block", ("long", 2)),
    ((1 << 22, 32, 1000.0, 64.0, 100.0), "sweep", ("long", 2)),
    ((1 << 23, 32, 1000.0, 64.0, 100.0), "sweep", ("long", 2)),
    ((1 << 24, 32, 1000.0, 0.5, 300.0), "sweep", ("long", 2)),
    ((1 << 22, 16, 1437.0, -64.0, -478.80), "block", ("long", 0)),
    ((1 << 24, 256, 1000.0, 0.05, 3000.0), "sweep", ("long", 1)),
    (CONFIG1, "block", ("long", 2)),
    (CONFIG2, "block", ("row16", "table")),
    (CONFIG2, "sweep", ("row16", "fly")),
    (CONFIG3, "block", ("bigrow", 5)),
    (CONFIG3, "sweep", ("bigrow", 3)),
    ((1 << 20, 1024, 1000.0, 500.0, 56.778), "sweep", ("unfused", None)),
    ((1 << 22, 4, 1000.0, 500.0, 56.778), "block", ("unfused", None)),
])
def test_variant_selection(geom, path, expect):
    assert chirp_variant(*geom, path) == expect


def test_config4_ladder_runs_two_newton_steps():
    for g in CONFIG4:
        assert chirp_variant(*g, "sweep") == ("long", 2) == chirp_variant(*g, "block"), g


def test_gpu_cases_reach_every_route_and_variant():
    assert gpu_case_pairs() == EXPECTED_PAIRS
    lengths = {ChirpParams(*c[1:]).L for c in GPU_CASES}
    assert set(ROW16) | set(BIGROW) | set(LONG) | {512, 1 << 19} <= lengths
    assert {long_geometry(L)[0] for L in LONG if L in lengths} == {256, 512}    # both first-sweep lengths


def test_fma_emulation_is_exact():
    """the emulated fma against exact rational arithmetic on the inputs a Newton step sees"""
    from fractions import Fraction
    rng = np.random.default_rng(7)
    f = 1000.0 + rng.random(200) * 500
    r = (1.0 / f) * (1 + rng.standard_normal(200) * 1e-9)
    inner = fma(-f, r, 1.0)
    outer = fma(r, inner, r)
    for i in range(200):
        assert inner[i] == float(Fraction(-f[i]) * Fraction(r[i]) + 1)
        assert outer[i] == float(Fraction(r[i]) * Fraction(inner[i]) + Fraction(r[i]))


PRODUCTION = ([("config1", CONFIG1, "block"), ("config3_sweep", CONFIG3, "sweep")] +
              [(f"config4_dm{g[-1]:g}", g, "sweep") for g in CONFIG4])


@pytest.mark.parametrize("name,geom,path", PRODUCTION, ids=[p[0] for p in PRODUCTION])
def test_newton_phase_error_within_design_bound(name, geom, path):
    """(a) at the production geometries the reciprocal chains the kernels walk keep the chirp phase within 1e-9 cycles
    of the exact one, plus a few ulp of |k| for the chain's own roundings: rows at both band edges and the middle"""
    route, variant = chirp_variant(*geom, path)
    assert (route, variant) in {("bigrow", 1), ("bigrow", 3), ("bigrow", 4), ("long", 1), ("long", 2)}
    p = ChirpParams(*geom)
    excess, worst, worst_ulps = -np.inf, 0.0, 0.0
    for row in sampled_rows(p.C):
        f, r = chain_reciprocals(p, route, variant, row)
        err, k = phase_error(p, f, r)
        excess = max(excess, float((err - ROUNDING_ULPS * EPS * k).max()))
        worst = max(worst, float(err.max()))
        worst_ulps = max(worst_ulps, float((err / np.maximum(EPS * k, 1e-300)).max()))
    print(f"{name}: {route} variant {variant}: largest phase error {worst:.2e} cycles, {worst_ulps:.2f} ulp of |k|")
    assert excess <= PHASE_BOUND


NEWTON_GPU_CASES = [c for c in GPU_CASES
                    if chirp_variant(*c[1:], "sweep") in {("bigrow", 3), ("bigrow", 4), ("long", 2)}]


@pytest.mark.parametrize("case", NEWTON_GPU_CASES, ids=[c[0] for c in NEWTON_GPU_CASES])
def test_a_dropped_newton_step_is_visible_at_the_gpu_geometries(case):
    """(b) at every GPU test geometry that runs two far Newton steps, one step fewer leaves an RMS phase error above
    2e-6 cycles (2 pi 2e-6 > 1e-5 rel-L2): the GPU comparison with float64 would fail. With both steps the RMS error
    stays three orders of magnitude below that."""
    route, variant = chirp_variant(*case[1:], "sweep")
    p = ChirpParams(*case[1:])
    sq, sq_full, count = 0.0, 0.0, 0
    for row in sampled_rows(p.C, 9):
        f, r = chain_reciprocals(p, route, variant, row, drop_far=1)
        err, _ = phase_error(p, f, r)
        sq += float((err ** 2).sum())
        f, r = chain_reciprocals(p, route, variant, row)
        sq_full += float((phase_error(p, f, r)[0] ** 2).sum())
        count += p.L
    rms, rms_full = np.sqrt(sq / count), np.sqrt(sq_full / count)
    print(f"{case[0]}: {route} variant {variant}: RMS phase error {rms_full:.2e} cycles, {rms:.2e} with a far step dropped")
    assert rms > DROPPED_STEP_RMS
    assert rms_full < 1e-3 * DROPPED_STEP_RMS
