"""CPU oracle of the waterfall thumbnail (simplify_spectrum_pipe_2, S/pipeline/spectrum_pipe.hpp:82-143): a serial
restatement in numpy float32 of resample_spectrum_3 with norm() (S/spectrum/simplify_spectrum.hpp:423-620),
simplify_spectrum_normalize_with_average_value (:627-644, map_average of S/algorithm/map_reduce.hpp) and
generate_pixmap (:700-731). Every fp32 operation is the reference's, one IEEE rounding each, in the reference's
order; the work-item splits (resample: nb_work_item per pixel; map_average: work-groups x work-items) are the ones the
reference computes for the host device of oracle/ref_shim (32 work-items, 8 compute units, sub-group size 32), so the
results are bit-identical to the reference run there (tests/golden/srtb_thumbnail_ref_vectors.npz).

Also the seeded test geometries shared by the golden generator and the tests."""
from __future__ import annotations

import numpy as np

F = np.float32
FLT_EPSILON = F(np.finfo(np.float32).eps)
COLOR_0, COLOR_1, COLOR_OVERFLOW = 0xFF1F1E33, 0xFF33E1F1, 0xFFE0E1CC

# host-shim device limits the reference's work-item split is computed from
_MAX_WORK_ITEM = 32  # min(max_work_group_size, max_work_item_sizes[0])
_LOCAL_MEM = 64 * 1024
_SUB_GROUP = 32
_COMPUTE_UNITS = 8


def extents(n_out: int, n_in: int):
    """per output index: (lo, hi, wl, wh) — cells [lo, hi) weight 1, cell lo - 1 weight wl (> 0 only), cell hi
    weight wh (> 0 only); the reference's fp32 edge expressions: i / out_f * in_f, ceil, floor"""
    i = np.arange(n_out, dtype=np.float64)
    a = (i.astype(F) / F(n_out)) * F(n_in)
    b = ((i + 1).astype(F) / F(n_out)) * F(n_in)
    lr, hr = np.ceil(a), np.floor(b)
    wl = np.where(lr > a, lr - a, F(0)).astype(F)
    wh = np.where(b > hr, b - hr, F(0)).astype(F)
    return lr.astype(np.int64), hr.astype(np.int64), wl, wh


def norm(spec: np.ndarray) -> np.ndarray:
    """|x|^2 = re * re + im * im in fp32 (S/math.hpp:59-66)"""
    s = np.ascontiguousarray(spec, dtype=np.complex64)
    re, im = s.real.astype(F), s.imag.astype(F)
    return re * re + im * im


def nb_work_item(in_width: int, out_width: int) -> int:
    required = max(int(np.round(F(in_width) / F(out_width))), 1)
    return min(_MAX_WORK_ITEM, _LOCAL_MEM // 4, required, _SUB_GROUP)


def resample(intensity: np.ndarray, out_width: int, out_height: int) -> np.ndarray:
    """resample_spectrum_3 on |x|^2 given as [in_height][in_width] float32"""
    p = np.ascontiguousarray(intensity, dtype=F)
    in_height, in_width = p.shape
    nb = nb_work_item(in_width, out_width)
    xlo, xhi, xwl, xwh = extents(out_width, in_width)
    ylo, yhi, ywl, ywh = extents(out_height, in_height)
    kmax = int(np.max(np.maximum(xhi - xlo, 0) + nb - 1) // nb) if out_width else 0
    j = np.arange(nb)
    lcell = np.maximum(xlo - 1, 0)
    hcell = np.minimum(xhi, in_width - 1)
    zero = F(0)

    def sample(y):  # [out_width][nb]: work item j's partial x sum of row y
        row = p[y]
        acc = np.zeros((out_width, nb), F)
        acc[:, 0] += np.where(xwl > 0, xwl * row[lcell], zero)
        for k in range(kmax):
            x = xlo[:, None] + j[None, :] + k * nb
            m = x < xhi[:, None]
            acc += np.where(m, row[np.where(m, x, 0)], zero)
        acc[:, nb - 1] += np.where(xwh > 0, xwh * row[hcell], zero)
        return acc

    out = np.empty((out_height, out_width), F)
    reduce_size = (1 << (nb - 1).bit_length()) >> 1
    for y2 in range(out_height):
        s = np.zeros((out_width, nb), F)
        if ywl[y2] > 0:
            s += ywl[y2] * sample(ylo[y2] - 1)
        for y in range(ylo[y2], yhi[y2]):
            s += sample(y)
        if ywh[y2] > 0:
            s += ywh[y2] * sample(yhi[y2])
        off = reduce_size
        while off > 0:  # work-items run in index order between barriers: each reads its partner's old value
            m = nb - off
            if m > 0:
                s[:, :m] = s[:, :m] + s[:, off:off + m]
            off >>= 1
        out[y2] = s[:, 0]
    return out


def average(x: np.ndarray) -> F:
    """map_average (sum / float(count)) with the SyclParallelSTL buffer_mapreduce split of the host shim"""
    v = np.ascontiguousarray(x, dtype=F).ravel()
    size = v.size
    nwi = min(_MAX_WORK_ITEM, _LOCAL_MEM // 4, size)
    nwg = min(_COMPUTE_UNITS, -(-size // nwi))
    per_wi = -(-size // (nwi * nwg))
    per_wg = per_wi * nwi
    nwg = max(1, -(-size // per_wg))
    total = F(0)
    for g in range(nwg):
        seg = v[g * per_wg:min((g + 1) * per_wg, size)]
        k = -(-seg.size // nwi)
        pad = np.zeros(k * nwi, F)
        pad[:seg.size] = seg
        rows = pad.reshape(k, nwi)
        acc = rows[0].copy()
        for r in range(1, k):  # padding zeros add nothing
            acc += rows[r]
        a = acc[0]
        for lane in range(1, min(nwi, seg.size)):
            a = F(a + acc[lane])
        total = F(total + a)
    return F(total / F(size))


def pixmap(v: np.ndarray, argb_0=COLOR_0, argb_1=COLOR_1, argb_overflow=COLOR_OVERFLOW) -> np.ndarray:
    """generate_pixmap: v in [0, 1] -> per ARGB channel (1 - v) * c0 + v * c1, truncated; else argb_overflow"""
    v = np.asarray(v, F)
    u = F(1) - v
    out = np.zeros(v.shape, np.uint32)
    for shift in (24, 16, 8, 0):
        c0 = F((argb_0 >> shift) & 0xFF)
        c1 = F((argb_1 >> shift) & 0xFF)
        ch = u * c0 + v * c1
        ok = (v >= 0) & (v <= 1)
        out |= (np.where(ok, ch, 0).astype(np.uint32) & 0xFF) << np.uint32(shift)
    return np.where((v >= 0) & (v <= 1), out, np.uint32(argb_overflow)).astype(np.uint32)


def simplify_spectrum(spec_or_norm: np.ndarray, out_width: int, out_height: int, argb_0=COLOR_0, argb_1=COLOR_1,
                      argb_overflow=COLOR_OVERFLOW):
    """(resampled intensity before scaling, average, normalised intensity, ARGB32 pixmap) of a [C][L] spectrum
    (complex64) or of its |x|^2 (float32)"""
    a = np.asarray(spec_or_norm)
    p = norm(a) if np.iscomplexobj(a) else a.astype(F)
    raw = resample(p, out_width, out_height)
    avg = average(raw)
    inten = raw.copy()
    if avg > FLT_EPSILON:
        inten *= F(1) / (avg * F(2))
    return raw, avg, inten, pixmap(inten, argb_0, argb_1, argb_overflow)


def unexplained_pixels(inten: np.ndarray, want: np.ndarray, got: np.ndarray, rel: float = 1e-5, argb_0=COLOR_0,
                       argb_1=COLOR_1, argb_overflow=COLOR_OVERFLOW):
    """(pixels that differ, pixels whose difference is not explained): a pixel's difference is explained when the
    oracle intensity v lies within `rel` (relative) of 1, or every differing ARGB channel differs by 1 and its exact
    value (1 - v) c0 + v c1 lies within rel * |v| * |c1 - c0| (plus fp32 rounding) of an integer step. A channel with
    c0 == c1 (alpha) sits on a step for every v, so its truncation may go either way on any pixel."""
    v = np.asarray(inten, np.float64)
    want, got = np.asarray(want, np.uint32), np.asarray(got, np.uint32)
    diff = want != got
    ok = np.abs(v - 1.0) <= rel
    in_range = (v >= 0) & (v <= 1)
    chan_ok = np.ones(v.shape, bool)
    for shift in (24, 16, 8, 0):
        c0 = float((argb_0 >> shift) & 0xFF)
        c1 = float((argb_1 >> shift) & 0xFF)
        cw, cg = (want >> shift) & 0xFF, (got >> shift) & 0xFF
        ch = (1.0 - v) * c0 + v * c1
        near = np.abs(ch - np.round(ch)) <= rel * np.abs(v) * abs(c1 - c0) + 1e-4
        step = np.abs(cw.astype(np.int64) - cg.astype(np.int64)) <= 1
        chan_ok &= (cw == cg) | (near & step & in_range)
    bad = diff & ~(ok | chan_ok)
    return int(diff.sum()), int(bad.sum())


# ---- seeded test geometries: name -> (C, L, H, W, kind)
CASES = {
    "nonint_down": (96, 1000, 40, 70, "noise"),
    "nonint_wide": (128, 2048, 60, 240, "noise"),
    "integer": (128, 1024, 32, 128, "noise"),
    "upsample": (24, 50, 64, 120, "noise"),
    "sk_zeroed": (64, 800, 20, 90, "zeroed"),
    "tiny_average": (48, 400, 16, 40, "tiny"),
    "impulse": (40, 300, 16, 50, "impulse"),
    "wide_ratio": (16, 8192, 8, 100, "noise"),
}


def case_spectrum(name: str) -> np.ndarray:
    """the [C][L] complex64 spectrum of a named case, from a fixed seed"""
    C, L, _, _, kind = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    if kind == "impulse":
        s = np.zeros((C, L), np.complex64)
        s[C // 3, L // 3 + 1] = 3 + 4j
        return s
    s = (rng.standard_normal((C, L)) + 1j * rng.standard_normal((C, L))).astype(np.complex64)
    s *= np.linspace(0.5, 2.0, C, dtype=np.float32)[:, None]  # a band shape
    if kind == "zeroed":
        s[[3, 4, 17, 40, 41, 42, 63]] = 0  # rows the spectral-kurtosis stage zaps
    if kind == "tiny":
        s *= np.float32(1e-5)  # |x|^2 ~ 1e-10: the average stays below FLT_EPSILON
    return s
