"""The s1, manual-range and spectral-kurtosis zap decisions of every block route against float64 (rfi_truth.py).

A block's dynamic spectrum carries its decisions: a channel row that SK zapped is all zero, and the forward FFT of a
kept row gives back coef L X chirp on every bin s1 kept and 0 on every bin it zapped (rfi_truth.recover_s1_mask). So
each case compares, against the float64 truth of the same samples:
- the s1 mask of every kept channel, bin by bin (bins with |X|^2 < 1e-6 mean cannot be told apart and are left out);
- the SK decision of every channel, the truth's SK formed from the GPU's own s1 mask on kept channels (so a border s1
  bin cannot move it) and, on zapped channels, accepted either way when flipping the channel's border s1 bins would
  move its SK across an edge;
- zero_count, against the float64 count of all-zero rows, give or take the channels whose SK lies on an edge;
- and, in one test, the kernels each case's block route and path launches (torch.profiler, in a fresh process), against
  the routes rfi_truth.rfi_route names for it.

Margins: an s1 decision may differ from float64 only within 1e-5 of the float64 limit (relative): |X|^2 of the fp32
R2C is good to about 2e-6 there. An SK decision may differ only within 1e-4 of the nearer window edge: the fp32 chirp
and waterfall FFT (rel-L2 <= 1e-5) move SK by up to about 2e-5. A route whose mean drops or double-counts a bin holding
1 % of the power, or whose window is off by a few 1e-3, flips decisions far outside these margins.

Informativeness: each route-matrix and multi-stream case must hold at least 100 s1 decisions within (1e-5, 1e-3] of
the limit and 10 SK decisions within (1e-4, 1e-2] of an edge (fewer where the block has fewer bins or channels than
that takes), so that a case whose thresholds drifted away from its data fails instead of passing vacuously. The SK
threshold of each case is set from the float64 SK of its own channels, putting the window's edges near their 20th and
80th percentiles.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import rfi_truth as rt  # noqa: E402
import srtb_b200  # noqa: E402
from test_fft_kernel_coverage import normalise  # noqa: E402
from test_gpu_parity import make_block_config  # noqa: E402
from test_rfi_truth import (RANGE_CASES, ROUTE_CASES, S1_MARGIN, SK_MARGIN, SPIKE_GEOMS, STREAM_CASES,  # noqa: E402
                            STREAM_FORMATS)

AVG_THR = 1.5           # the J1644 setting: about 22 % of the noise bins lie above 1.5 x the mean
D_E6 = 4.148808e3 * 1e6


@pytest.fixture(scope="module")
def rctx():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    torch.cuda.set_device(0)
    c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _free_memory():
    yield
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------- kernels a route launches
MEAN_KERNELS = {"post": "r2c_post_kernel", "fixup2": "r2c_col0_fixup_kernel", "fixup3": "r2c_col0_fixup_kernel",
                "fixup4": "r2c_col0_fixup_kernel", "rows_split": "r2c_rows_split_kernel"}
S1_KERNELS = {"row16": {"fft_row16_tma_kernel"}, "bigrow": {"fft_bigrow_kernel", "waterfall_sweep_order_kernel"},
              "long": {"fft_col16_tma_kernel", "fft_col_tma_kernel"}, "unfused": {"dedisperse_kernel"}}
SK_KERNELS = {"row16": {"fft_row16_tma_kernel"}, "row8_512": {"fft_row_tma_kernel"},
              "bigrow": {"fft_bigrow_kernel", "waterfall_sweep_order_kernel"}, "long": {"sk_decide_kernel"},
              "unfused": {"sk_kernel"}}


def profiled(call, tries=4):
    """(call(), base names of the CUDA kernels it launched). The window is bracketed by one torch kernel on each side;
    torch.profiler now and then loses the start of a window, so a window without both brackets is discarded and the
    call (deterministic: nothing but its outputs changes) is run again in a new one"""
    from torch.profiler import ProfilerActivity, profile
    mark = torch.zeros(1, device="cuda")
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            mark.add_(1)
            out = call()
            mark.add_(1)
            torch.cuda.synchronize()
        events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if sum("at::native" in e for e in events) >= 2:
            return out, {normalise(e).split("<")[0].split("::")[-1] for e in events}
    raise AssertionError("torch.profiler recorded no complete window in a fresh process")


def check_route(label, names, route):
    (mean, first), s1, sk = route
    assert MEAN_KERNELS[mean] in names, f"{label}: {mean} route did not launch {MEAN_KERNELS[mean]}"
    unpack = any(n.startswith("unpack_") for n in names)
    assert unpack == (first == "unpacked"), f"{label}: first sweep {first}, launched {sorted(names)}"
    assert S1_KERNELS[s1] & names, f"{label}: s1 route {s1} launched none of {S1_KERNELS[s1]}"
    assert SK_KERNELS[sk] & names, f"{label}: SK route {sk} launched none of {SK_KERNELS[sk]}"


# ----------------------------------------------------------------------------- float64 truth on the device
def device_spectrum(ptr, C_, L):
    """a torch copy [C][L] complex64 of the dynamic spectrum at a raw device pointer"""
    cudart = C.CDLL("libcudart.so")
    cudart.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    out = torch.empty(C_ * L, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    assert cudart.cudaMemcpy(out.data_ptr(), ptr, out.numel() * 8, 3) == 0
    return out.view(C_, L)


class Truth:
    """float64 truth of one stream: its R2C, s1 mask (manual ranges included), limit and the chirp of a DM"""

    def __init__(self, samples, cfg, bins=()):
        n = cfg.baseband_input_count
        self.nc = n // 2
        self.C = min(cfg.spectrum_channel_count, self.nc)
        self.L = self.nc // self.C
        self.cfg = cfg
        Xf = torch.fft.rfft(torch.as_tensor(samples).cuda().to(torch.float64))
        self.nyquist_power = float(Xf[self.nc].abs() ** 2)
        self.X = Xf[:self.nc].contiguous()
        del Xf
        self.mask, self.limit, self.pw = rt.s1_truth(self.X, cfg.mitigate_rfi_average_method_threshold, bins)
        self.mean = float(self.pw.mean())
        self.manual = torch.zeros(self.nc, dtype=torch.bool, device="cuda")
        for lo, hi in bins:
            self.manual[lo:hi + 1] = True
        self.coef = float(srtb_b200.norm_coefficient(self.nc, cfg.spectrum_channel_count))

    def chirp(self, dm):
        f_min, bw = np.float32(self.cfg.baseband_freq_low), np.float32(self.cfg.baseband_bandwidth)
        f_c = float(np.float32(f_min + bw))
        df = float(np.float32(bw / np.float32(self.nc)))
        f = float(f_min) + df * torch.arange(self.nc, dtype=torch.float64, device="cuda")
        k = D_E6 * float(np.float32(dm)) / f * ((f - f_c) / f_c) ** 2
        ang = -2 * np.pi * (k - torch.trunc(k))
        return torch.polar(torch.ones_like(ang), ang)

    def sk(self, mask, dm, rows=None):
        """float64 SK of the channel rows (all, or the indices `rows`) with the bins of `mask` [C][L] zapped"""
        X = self.X.view(self.C, self.L)
        ch = self.chirp(dm).view(self.C, self.L)
        if rows is not None:
            X, ch, mask = X[rows], ch[rows], mask[rows]
        Z = torch.where(mask, 0, X * self.coef) * ch
        return rt.sk_truth(torch.fft.ifft(Z, dim=-1))

    def sk_thr(self, dm):
        """the threshold whose window edges sit near the 20th and 80th percentiles of the float64 SK of this stream"""
        sk = self.sk(self.mask.view(self.C, self.L), dm)
        sk = sk[~torch.isnan(sk)].cpu().numpy()
        f = (np.float32(self.L) - 1) / (np.float32(self.L) + 1)
        q20, q80 = np.percentile(sk, [20, 80])
        return float(1 + (q80 - q20) / (2 * f))


def check_stream(label, res, gspec, t, dm, sk_thr, need_s1=0, need_sk=0):
    """one stream's decisions against its float64 truth; prints and returns the counts"""
    C_, L = t.C, t.L
    gzero = (gspec == 0).all(dim=1)
    keep = ~gzero
    X = t.X.view(C_, L)
    # s1 and the manual ranges, bin by bin, on every kept channel
    if not bool(keep.any()):
        keep[0] = True              # an all-zero block: one row keeps the shapes; its recovered mask is all zapped
    zapped, amb = rt.recover_s1_mask(gspec[keep], X[keep], t.coef, t.mean)
    tmask = t.mask.view(C_, L)[keep]
    stat = torch.where(t.manual.view(C_, L)[keep], float("inf"), t.pw.view(C_, L)[keep])
    ok = ~amb
    d1 = rt.compare_decisions(zapped[ok], stat[ok], t.limit, S1_MARGIN, truth=tmask[ok])
    assert d1.worst <= S1_MARGIN, f"{label}: {d1.flips} s1 flips, one {d1.worst:.2e} from the limit"
    # SK, every channel: the GPU's s1 mask where it can be read back
    m = t.mask.view(C_, L).clone()
    m[keep] = torch.where(amb, tmask, zapped)
    sk = t.sk(m, dm)
    lo, hi = rt.sk_window(sk_thr, L)
    nan = torch.isnan(sk)
    got = gzero & ~nan
    truth = rt.truth_decisions(sk, (lo, hi))
    dist = rt.decision_distance(sk, (lo, hi))
    flips = torch.nonzero(got != truth).flatten().tolist()
    alt_ok = 0
    if flips:
        border = (rt.decision_distance(t.pw.view(C_, L), t.limit) <= S1_MARGIN) & ~t.manual.view(C_, L)
        for c in flips:
            if dist[c] <= SK_MARGIN or not bool(got[c]) or not bool(border[c].any()):
                continue
            alt = m.clone()
            alt[c] ^= border[c]
            if bool(rt.truth_decisions(t.sk(alt, dm, [c]), (lo, hi))[0]) == bool(got[c]):
                alt_ok += 1
                dist[c] = 0.0
    d2 = rt.compare_decisions(got, sk, (lo, hi), SK_MARGIN, truth=truth)
    worst = max([float(dist[c]) for c in flips] + [0.0])
    assert worst <= SK_MARGIN, f"{label}: {d2.flips} SK flips, one {worst:.2e} from the window [{lo:.6f}, {hi:.6f}]"
    # zero_count: the all-zero rows of the float64 chain, up to the channels on an edge
    expect_zero = int((truth | nan).sum())
    slack = int((dist <= SK_MARGIN).sum()) + alt_ok
    assert abs(int(res.zero_count) - expect_zero) <= slack, f"{label}: zero_count {res.zero_count}, truth {expect_zero}"
    print(f"{label}: s1 {d1.total} bins ({int(amb.sum())} ambiguous), {int(zapped.sum())} zapped, {d1.flips} flips "
          f"(worst {d1.worst:.1e}), {d1.informative} informative; SK window [{lo:.5f}, {hi:.5f}] on {C_} channels: "
          f"{int(got.sum())} zapped, {int(nan.sum())} all-zero inputs, {d2.flips} flips (worst {worst:.1e}, "
          f"{alt_ok} by border s1 bins), {d2.informative} informative; zero_count {res.zero_count}")
    assert d1.informative >= need_s1, f"{label}: {d1.informative} informative s1 decisions (< {need_s1})"
    assert d2.informative >= need_sk, f"{label}: {d2.informative} informative SK decisions (< {need_sk})"
    return d1, d2


def needs(t):
    """the informativeness floor: 100 s1 and 10 SK decisions, or what a block of this many bins and channels holds
    (about 6.6e-4 Nc bins lie within (1e-5, 1e-3] of the limit at avg_thr 1.5)"""
    return min(100, t.nc // 4096), min(10, t.C // 8)


def straddling_bins(n, C_, f_low, bw):
    """a manual range (MHz) around the first bin of channel row C/2: 40 bins either side, or 8 float32 ulp of the
    frequency where the band is so narrow that 40 bins are less"""
    nc = n // 2
    L = nc // C_
    df = bw / nc
    f_edge = f_low + df * (C_ // 2) * L
    half = max(40 * abs(df), 8 * float(np.spacing(np.float32(f_edge))))
    pair = (f_edge - half, f_edge + half)
    bins = srtb_b200.rfi_range_to_bins(pair[0], pair[1], f_low, bw, nc)
    assert bins is not None and bins[0] < (C_ // 2) * L <= bins[1]
    return [pair], [bins]


def noise(n, seed, bits=-8, sigma=rt.SIGMA):
    if bits == -16:
        rng = np.random.default_rng(seed)
        return np.round(rng.standard_normal(n, np.float32) * 300).astype(np.int16)
    return rt.noise_int8(n, seed, sigma)


# ----------------------------------------------------------------------------- A. the route matrix
@pytest.mark.parametrize("case", ROUTE_CASES, ids=[c[0] for c in ROUTE_CASES])
def test_route_decisions_vs_float64(rctx, case):
    """process_block and the last trial of a two-trial DM sweep, every decision against float64"""
    name, n, C_, f_low, bw, dm, bits = case
    L = n // 2 // C_
    samples = noise(n, 1000 + ROUTE_CASES.index(case), bits)
    pairs, bins = straddling_bins(n, C_, f_low, bw)
    cfg = make_block_config(n, bits, srtb_b200.FORMAT_SIMPLE, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                            avg_thr=AVG_THR, sk_thr=1.05, snr=50.0, pairs=pairs)
    t = Truth(samples, cfg, bins)
    thr = t.sk_thr(dm)
    cfg.mitigate_rfi_spectral_kurtosis_threshold = thr
    d = torch.from_numpy(samples.view(np.uint8)).cuda()
    need_s1, need_sk = needs(t)
    res = rctx.process_block(cfg, d, d.numel(), None, on_device=True)[0]
    route = rt.rfi_route(n, C_, bits, rt.SIMPLE, "block")
    check_stream(f"{name} block {route}", res, device_spectrum(rctx.block_spectrum_ptr(0), C_, L), t, dm, thr,
                 need_s1, need_sk)
    dm_a = 0.5 * dm if dm else 100.0
    res = rctx.process_block_dm_sweep(cfg, d, d.numel(), [dm_a, dm], on_device=True)[1][0]
    route = rt.rfi_route(n, C_, bits, rt.SIMPLE, "sweep")
    check_stream(f"{name} sweep {route}", res, device_spectrum(rctx.sweep_spectrum_ptr(), C_, L), t, dm, thr,
                 need_s1, need_sk)


# ----------------------------------------------------------------------------- B. bins with special treatment
_NOISE = {}


@pytest.mark.parametrize("kind", rt.SPIKES)
@pytest.mark.parametrize("route", list(SPIKE_GEOMS))
def test_special_bins_in_the_mean(rctx, route, kind):
    """one spike of 1 - 5 % of the block's power in DC, M / 2, column 0 of the fused split, a generic bin or the
    Nyquist bin (which must not count): the limit, and so every s1 decision, follows the float64 mean"""
    n, C_ = SPIKE_GEOMS[route]
    L = n // 2 // C_
    if route not in _NOISE:
        _NOISE.clear()
        _NOISE[route] = rt.noise_int8(n, 40)
    samples = rt.with_spike(_NOISE[route], kind)
    dm = 56.778
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, dm, fs=1e9, avg_thr=AVG_THR, sk_thr=1.05, snr=50.0)
    t = Truth(samples, cfg)
    k = rt.spike_bin(n, kind)
    total = float(t.pw.sum())
    frac = (t.nyquist_power if kind == "nyquist" else float(t.pw[k])) / total
    assert 0.01 <= frac <= 0.05, f"bin {k} holds {frac:.4f} of the power"
    thr = t.sk_thr(dm)
    cfg.mitigate_rfi_spectral_kurtosis_threshold = thr
    d = torch.from_numpy(samples.view(np.uint8)).cuda()
    res = rctx.process_block(cfg, d, n, None, on_device=True)[0]
    check_stream(f"{route} {kind} (bin {k}, {100 * frac:.1f} % of the power)", res,
                 device_spectrum(rctx.block_spectrum_ptr(0), C_, L), t, dm, thr)


# ----------------------------------------------------------------------------- C. streams of unequal power
def _interleave(fmt, a, b):
    raw = np.empty(2 * a.size, np.int8)
    if fmt == "naocpsr_snap1":
        raw.reshape(-1, 4)[:, 0:2] = a.reshape(-1, 2)
        raw.reshape(-1, 4)[:, 2:4] = b.reshape(-1, 2)
    elif fmt == "interleaved_samples_2":
        raw[0::2], raw[1::2] = a, b
    else:                                               # gznupsr_a1: words of four samples alternate
        raw.reshape(-1, 2, 4)[:, 0] = a.reshape(-1, 4)
        raw.reshape(-1, 2, 4)[:, 1] = b.reshape(-1, 4)
    return raw


@pytest.mark.parametrize("case", STREAM_CASES, ids=[c[0] for c in STREAM_CASES])
def test_unequal_streams_each_use_their_own_mean(rctx, oracle, case):
    """stream 1 at 3 x the noise sigma of stream 0 (9 x the mean): process_block (two lanes), the ring and the DM
    sweep's best-trial re-run (which restores each stream's mean) decide every stream against its own truth"""
    name, n, C_, fmt, f_low, bw, dm = case
    L = n // 2 // C_
    bits = 8 if fmt == "gznupsr_a1" else -8
    a = rt.noise_int8(n, 70, 10.0)
    b = rt.noise_int8(n, 71, 30.0)
    raw = _interleave(fmt, a, b)
    if fmt == "naocpsr_snap1":
        samples = oracle.unpack_snap1(raw.view(np.uint8), n)
    elif fmt == "interleaved_samples_2":
        samples = oracle.unpack_interleaved_2(raw.view(np.uint8), n, bits)
    else:
        samples = oracle.unpack_gznupsr_a1(raw, n, 2)
    assert np.array_equal(samples[0], a) and np.array_equal(samples[1], b)
    pairs, bins = straddling_bins(n, C_, f_low, bw)
    cfg = make_block_config(n, bits, STREAM_FORMATS[fmt], C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                            avg_thr=AVG_THR, sk_thr=1.05, snr=50.0, pairs=pairs)
    truths = [Truth(s, cfg, bins) for s in samples]
    assert truths[1].mean > 8 * truths[0].mean
    thr = truths[0].sk_thr(dm)
    cfg.mitigate_rfi_spectral_kurtosis_threshold = thr
    need_s1, need_sk = needs(truths[0])
    pinned = torch.from_numpy(raw.view(np.uint8).copy()).pin_memory()
    res = rctx.process_block(cfg, pinned, raw.size, None)
    route = rt.rfi_route(n, C_, bits, STREAM_FORMATS[fmt], "block")
    for s in range(2):
        check_stream(f"{name} block stream {s} {route}", res[s], device_spectrum(rctx.block_spectrum_ptr(s), C_, L),
                     truths[s], dm, thr, need_s1, need_sk)
    ticket = rctx.submit_block(cfg, pinned, raw.size)
    res, _, specs = rctx.collect_block_ex(ticket)
    for s in range(2):
        check_stream(f"{name} ring stream {s}", res[s], device_spectrum(specs[s], C_, L), truths[s], dm, thr)
    dms = [0.5 * dm, dm]
    results, _, best, _, spec = rctx.process_block_dm_sweep(cfg, pinned, raw.size, dms, outputs=True)
    for s in range(2):
        got = spec[s][:n].view(torch.complex64).view(C_, L)
        check_stream(f"{name} sweep stream {s}, best trial {best[s]}", results[best[s]][s], got, truths[s],
                     dms[best[s]], thr)


# ----------------------------------------------------------------------------- D. manual ranges, linear layout
def manual_ranges(n, C_, f_low, bw):
    """(pairs in MHz, the bins the library zeroes, the RFI tone's bin): 19 ranges that convert, so that two zeroing
    launches run, plus an out-of-band pair and one above the band that do not. They cover bin 0 and bin Nc - 1, single
    bins, two overlapping ranges, a reversed pair, a whole channel (channel 11) and a range holding a strong tone"""
    nc = n // 2
    L = nc // C_
    b = [(0, 5), (nc - 7, nc - 1), (3 * L + 100, 3 * L + 100), (5 * L + 7, 5 * L + 7), (7 * L + 10, 7 * L + 60),
         (7 * L + 40, 7 * L + 90), (9 * L + 20, 9 * L + 30), (11 * L - 8, 12 * L + 7), (13 * L + 10, 13 * L + 60)]
    b += [(i * L + 33, i * L + 33 + i) for i in range(15, 25)]
    f = lambda k: f_low + bw * k / (nc - 1)                          # noqa: E731  (rfi_range_to_bins inverted)
    pairs = [(f(lo), f(hi)) for lo, hi in b]
    pairs[6] = pairs[6][::-1]                                        # reversed
    pairs.insert(4, (f(-3000), f(-1000)))                            # below the band
    pairs.append((f(nc + 1000), f(nc + 3000)))                       # above it
    conv = [srtb_b200.rfi_range_to_bins(p[0], p[1], f_low, bw, nc) for p in pairs]
    bins = [c for c in conv if c is not None]
    assert len(bins) == 19 and conv[4] is None and conv[-1] is None
    return pairs, bins, 13 * L + 35


@pytest.mark.parametrize("case", RANGE_CASES, ids=[c[0] for c in RANGE_CASES])
def test_manual_ranges_vs_float64(rctx, case):
    """every range zeroes its bins on process_block and on the last trial of a DM sweep; the tone inside a range
    (about 5 % of the power) still counts in the mean; the channel inside a range has NaN SK, is kept, and counts
    in zero_count"""
    name, n, C_, f_low, bw, dm = case
    L = n // 2 // C_
    pairs, bins, tone = manual_ranges(n, C_, f_low, bw)
    g = int(np.gcd(n, tone))
    t_ = np.arange(n // g)
    pattern = np.resize(np.round(6.5 * np.cos(2 * np.pi * ((tone // g) * t_ % (n // g)) / (n // g))), n)
    samples = np.clip(noise(n, 90).astype(np.int16) + pattern.astype(np.int16), -128, 127).astype(np.int8)
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                            avg_thr=AVG_THR, sk_thr=1.05, snr=50.0, pairs=pairs)
    t = Truth(samples, cfg, bins)
    frac = float(t.pw[tone]) / float(t.pw.sum())
    assert 0.03 < frac < 0.08, frac
    thr = t.sk_thr(dm)
    cfg.mitigate_rfi_spectral_kurtosis_threshold = thr
    d = torch.from_numpy(samples.view(np.uint8)).cuda()
    res = rctx.process_block(cfg, d, n, None, on_device=True)[0]
    spec = device_spectrum(rctx.block_spectrum_ptr(0), C_, L)
    assert not spec[11].any()
    route = rt.rfi_route(n, C_, -8, rt.SIMPLE, "block")
    check_stream(f"{name} block {route}", res, spec, t, dm, thr)
    res = rctx.process_block_dm_sweep(cfg, d, n, [0.5 * dm, dm], on_device=True)[1][0]
    check_stream(f"{name} sweep", res, device_spectrum(rctx.sweep_spectrum_ptr(), C_, L), t, dm, thr)


# ----------------------------------------------------------------------------- E. window branches, degenerate blocks
@pytest.mark.parametrize("label,n,C_,f_low,bw,dm,sk_thr,reserve", [
    ("swapped_window_0.97", 1 << 20, 512, 1000.0, 500.0, 56.778, 0.97, 0),
    ("upper_edge_only_2.5", 1 << 20, 64, 1000.0, 500.0, 56.778, 2.5, 0),
    ("reserved_tail_long", 1 << 22, 64, 1000.0, 64.0, 1.0, None, 1),
])
def test_window_branches(rctx, label, n, C_, f_low, bw, dm, sk_thr, reserve):
    """sk_thr < 1 (sk_bounds swaps the edges), sk_thr > 2 (the lower edge lies below any SK) and reserve_sample on
    with a reserved tail of thousands of samples per row (SK still spans all L samples)"""
    L = n // 2 // C_
    samples = noise(n, 120)
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                            avg_thr=AVG_THR, sk_thr=1.05, snr=50.0)
    cfg.baseband_reserve_sample = reserve
    if reserve:
        per_row = srtb_b200.nsamps_reserved(n, C_, f_low, bw, 2e6 * abs(bw), dm, 1) // C_
        assert 1000 < per_row < L // 4, per_row
    t = Truth(samples, cfg)
    thr = t.sk_thr(dm) if sk_thr is None else sk_thr
    cfg.mitigate_rfi_spectral_kurtosis_threshold = thr
    d = torch.from_numpy(samples.view(np.uint8)).cuda()
    res = rctx.process_block(cfg, d, n, None, on_device=True)[0]
    _, d2 = check_stream(label, res, device_spectrum(rctx.block_spectrum_ptr(0), C_, L), t, dm, thr)
    if sk_thr is not None and sk_thr < 1:
        assert 0 < res.zero_count < C_


def test_all_zero_block(rctx):
    """nothing is zapped, every SK is NaN, zero_count = C and detection is off"""
    n, C_ = 1 << 20, 512
    L = n // 2 // C_
    samples = np.zeros(n, np.int8)
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, 56.778, avg_thr=AVG_THR, sk_thr=1.05, snr=50.0)
    t = Truth(samples, cfg)
    assert t.limit == 0 and not bool(t.mask.any())
    d = torch.from_numpy(samples.view(np.uint8)).cuda()
    for path in ("block", "sweep"):
        if path == "block":
            res = rctx.process_block(cfg, d, n, None, on_device=True)[0]
            spec = device_spectrum(rctx.block_spectrum_ptr(0), C_, L)
        else:
            res = rctx.process_block_dm_sweep(cfg, d, n, [0.0, 56.778], on_device=True)[1][0]
            spec = device_spectrum(rctx.sweep_spectrum_ptr(), C_, L)
        assert not spec.any()
        assert res.zero_count == C_ and res.detect_enabled == 0
        assert bool(torch.isnan(t.sk(t.mask.view(C_, L), 56.778)).all())
        check_stream(f"all-zero block, {path}", res, spec, t, 56.778, 1.05)



# ----------------------------------------------------------------------------- the kernels of every route
def route_probes():
    """(label, n, C, bits, format, f_low, bw, dm, path) of every block route and path the cases above run"""
    out = [(f"{c[0]} {path}", c[1], c[2], c[6], srtb_b200.FORMAT_SIMPLE) + c[3:6] + (path,)
           for c in ROUTE_CASES for path in ("block", "sweep")]
    out += [(f"spikes {route}", n, C_, -8, srtb_b200.FORMAT_SIMPLE, 1000.0, 500.0, 56.778, "block")
            for route, (n, C_) in SPIKE_GEOMS.items()]
    out += [(f"{c[0]} {path}", c[1], c[2], 8 if c[3] == "gznupsr_a1" else -8, STREAM_FORMATS[c[3]]) + c[4:7] + (path,)
            for c in STREAM_CASES for path in ("block", "sweep")]
    return out


def probe_routes():
    """run in a fresh process (torch.profiler's state there is clean): every probe once on random bytes, printing one
    JSON line per probe with the kernels it launched"""
    import json
    torch.cuda.set_device(0)
    ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(7)
    for label, n, C_, bits, fmt, f_low, bw, dm, path in route_probes():
        nbytes = n * srtb_b200.FORMAT_STREAMS[fmt] * abs(bits) // 8
        d = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
        cfg = make_block_config(n, bits, fmt, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw), avg_thr=AVG_THR,
                                sk_thr=1.05, snr=50.0)
        if path == "block":
            _, names = profiled(lambda: ctx.process_block(cfg, d, nbytes, None, on_device=True))
        else:
            _, names = profiled(lambda: ctx.process_block_dm_sweep(cfg, d, nbytes, [0.5 * dm, dm], on_device=True))
        print(json.dumps([label, sorted(names)]), flush=True)
        del d
        torch.cuda.empty_cache()
    ctx.close()


def test_every_case_launched_its_routes():
    """each block route and path of the cases above launches the kernels rfi_route names for it: the mean's kernel,
    the unpack kernel exactly when the first sweep is not raw, and the kernels that apply s1 and decide SK. Profiled
    in a fresh process, because torch.profiler stops recording in a process that has opened many profiler windows
    (the GPU suite opens hundreds before this module)."""
    import json
    import os
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([str(root / "tests"), str(root / "simple-radio-telescope-backend_b200"),
                                         env.get("PYTHONPATH", "")])
    out = subprocess.run([sys.executable, "-c", "import test_gpu_rfi_decisions as m; m.probe_routes()"], env=env,
                         cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    got = dict(json.loads(line) for line in out.stdout.splitlines() if line.startswith("["))
    probes = route_probes()
    assert set(got) == {p[0] for p in probes}
    for label, n, C_, bits, fmt, *_, path in probes:
        route = rt.rfi_route(n, C_, bits, fmt, path)
        check_route(label, set(got[label]), route)
        print(f"{label}: {route}")
