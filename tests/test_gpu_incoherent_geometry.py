"""The semi-coherent DM search (srtb_b200_incoherent_dm_search) on the GPU at the geometry the executable runs it at:
config #3's stream shape (C = 2048, L = 16384) with trial lists whose groups are cut by count and by spread, single-trial
groups, group spreads on both sides of the 48 KiB shared-memory limit, a zero-filled last tile, series longer than
65535 tiles, and the executable's block seam. tests/incoherent_cases.py holds the cases and tests/test_incoherent_groups.py
checks on the CPU that each reaches the structure it is named for.

Truth is float64: tests/incoherent_oracle.py's definition, the channel sums formed on the device in float64. Tolerances
come from a bound, not from constants. The kernel forms v[j] = sum_c p_c with p_c = fl(fl(re^2) + fl(im^2)) >= 0, added
in fp32 in channel order, so |v32[j] - v64[j]| <= gamma_(C+1) v64[j], gamma_n = n u / (1 - n u), u = 2^-24 (Higham,
recursive summation, plus gamma_2 for each power). _bounds() carries that bound through the detector's own rounding (the
float mean, the fp64 scan stored as float, the boxcar differences, the fp64 sums of squares) to a bound on every boxcar
sample, the variance, the threshold and the peak S/N; a sample within its bound of the threshold may count either way,
and the peak index must be one whose value is within the bounds of the maximum."""
import resource
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import incoherent_cases as ic  # noqa: E402
import incoherent_grouping as ig  # noqa: E402
import incoherent_oracle as io  # noqa: E402
import srtb_b200  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

SNR, CHAN_THR, MAXBOX = 6.0, 0.9, 64
ZERO_CHANNELS = (3, 17, 40)
U, U64 = 2.0 ** -24, 2.0 ** -53
CASES = ic.cases()


def _gamma(n, u=U):
    return n * u / (1 - n * u)


def _spectrum(C_, L, seed):
    """complex64 [C][L] noise on the device as float32 [C][L][2], channels ZERO_CHANNELS flagged (all zero)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((C_, L, 2), device="cuda", generator=g, dtype=torch.float32)
    x[[c for c in ZERO_CHANNELS if c < C_]] = 0
    return x


def _plant(x, s, sm, k, t, amp):
    """a pulse along trial k's curve at series index t: amp added to the real part of x[c][t + S- + s[k][c]]"""
    C_ = x.shape[0]
    cols = torch.as_tensor(t + sm + s[k], device="cuda")
    rows = torch.arange(C_, device="cuda")
    keep = torch.ones(C_, dtype=torch.bool, device="cuda")
    keep[[c for c in ZERO_CHANNELS if c < C_]] = False
    x[rows[keep], cols[keep], 0] += amp


def _truth(x, s, sm, T):
    """v64 [n_dm][T] (numpy) and the zero count, from the float64 power of the device spectrum"""
    P = x.double().pow(2).sum(-1)
    j = torch.arange(T, device="cuda")
    v = torch.empty((s.shape[0], T), dtype=torch.float64, device="cuda")
    for d in range(s.shape[0]):
        idx = torch.as_tensor(s[d] + sm, device="cuda")[:, None] + j[None, :]
        v[d] = P.gather(1, idx).sum(0)
    zc = int((P[:, 0] == 0).sum())
    del P
    return v.cpu().numpy(), zc


def _bounds(v, C_, want):
    """per boxcar of io.detect's `want`: e[j] >= |sb32[j] - sb64[j]|, and bounds on the variance and threshold"""
    T = len(v)
    E = _gamma(C_ + 1) * v                           # the fp32 channel sum
    m = v.sum() / T
    em = E.mean() + _gamma(T, U64) * np.abs(v).mean() + 4 * U * abs(m)  # fp64 sum, float total, float T, division
    d = want["series"][0] if want["n_boxcars"] else v - m
    e1 = (1 + U) * (E + em) + U * np.abs(d)           # d32 = fl(v32 - m32)
    acc = np.cumsum(d)
    e_scan = _gamma(T, U64) * np.abs(d).sum() + 1e-300  # the fp64 running sum
    ce = np.concatenate([[0.0], np.cumsum(e1)])
    out = []
    for nb, b in enumerate(want["boxcar_length"]):
        sb = want["series"][nb]
        n = len(sb)
        if b == 1:
            e = e1
        else:  # fl(acc32[j + b] - acc32[j]), acc32 = fl(fp64 running sum of d32)
            win = ce[b + 1:T + 1] - ce[1:T - b + 1]
            e = (1 + 4 * U) * (win + 2 * e_scan + U * (np.abs(acc[b:]) + np.abs(acc[:T - b])) + U * np.abs(sb))
        var = want["variance"][nb]
        dsq = (2 * np.abs(sb) * e + e * e).sum() + _gamma(n, U64) * ((np.abs(sb) + e) ** 2).sum()
        dv = dsq / n + 5 * U * (var + dsq / n)
        thr_lo = SNR * np.sqrt(max(var - dv, 0.0)) * (1 - 3 * U)
        thr_hi = SNR * np.sqrt(var + dv) * (1 + 3 * U)
        out.append({"e": e, "var": (var - dv, var + dv), "thr": (thr_lo, thr_hi)})
    return out


def _check_trial(got, psnr, pidx, v, zc, C_, where, h_series=None, maxbox=MAXBOX):
    """one trial's header, peaks and (optionally) positive series against float64 within the bound; returns the truth"""
    want = io.detect(v, zc, C_, SNR, CHAN_THR, maxbox)
    assert got.zero_count == want["zero_count"], where
    assert bool(got.detect_enabled) == want["detect_enabled"], where
    assert got.n_boxcars == want["n_boxcars"], where
    assert got.time_series_count == want["time_series_count"] == len(v), where
    for nb, bd in enumerate(_bounds(v, C_, want)):
        sb, e = want["series"][nb], bd["e"]
        w = (where, nb)
        assert got.boxcar_length[nb] == want["boxcar_length"][nb], w
        assert got.series_length[nb] == want["series_length"][nb], w
        assert bd["var"][0] <= got.variance[nb] <= bd["var"][1], (w, got.variance[nb], want["variance"][nb], bd["var"])
        assert bd["thr"][0] <= got.threshold[nb] <= bd["thr"][1], (w, got.threshold[nb], bd["thr"])
        above, maybe = np.count_nonzero(sb - e > bd["thr"][1]), np.count_nonzero((sb + e > bd["thr"][0]) &
                                                                                 (sb - e <= bd["thr"][1]))
        assert above <= int(got.signal_count[nb]) <= above + maybe, (w, got.signal_count[nb], above, maybe)
        hi, lo = float(np.max(sb + e)), float(np.max(sb - e))
        p_hi = hi / np.sqrt(bd["var"][0]) * (1 + 4 * U)
        p_lo = lo / np.sqrt(bd["var"][1]) * (1 - 4 * U)
        assert p_lo <= psnr[nb] <= p_hi, (w, psnr[nb], p_lo, p_hi)
        cand = np.flatnonzero(sb + e >= lo)
        assert int(pidx[nb]) in cand, (w, int(pidx[nb]), cand[:8])
        if h_series is not None and got.signal_count[nb] > 0:
            assert np.all(np.abs(h_series[nb, :len(sb)].astype(np.float64) - sb) <= e), w
    return want


def _search(ctx, x, case, dms=None, h_series=None):
    fl, bw = ic.BANDS[case["band"]]
    dms = case["dms"] if dms is None else dms
    return ctx.incoherent_dm_search(x, case["time_count"], ic.C, case["reserved"], fl, bw, ic.SR, ic.DM, dms, SNR,
                                    CHAN_THR, MAXBOX, h_series)


def _geometry(case):
    fl, bw = ic.BANDS[case["band"]]
    s, sp, sm = io.shifts(ic.C, fl, bw, ic.SR, ic.DM, case["dms"])
    return s, sm, case["time_count"] - case["reserved"] - sp - sm


def _check_all(ctx, x, case, out=None):
    """the search of `case` on x (or its given result) against float64, every trial; returns (result, v64)"""
    s, sm, T = _geometry(case)
    res, (psnr, pidx), best, hs = _search(ctx, x, case) if out is None else out
    v, zc = _truth(x, s, sm, T)
    for d in range(len(case["dms"])):
        _check_trial(res[d], psnr[d], pidx[d], v[d], zc, ic.C, d, hs if d == best else None)
    return (res, (psnr, pidx), best, hs), v


def _chosen(case):
    """sorted slots -> trials: the first and last of every group cut by spread, every single-trial group, and dm"""
    s, _, _ = _geometry(case)
    order, groups, _, _, _ = ig.groups(s, case["dms"])
    pick = []
    for i, (first, count) in enumerate(groups):
        rows = s[order[first:first + count + 1]]
        cut = first + count < len(order) and int((rows.max(0) - rows.min(0)).max()) > ig.INC_SPREAD_MAX
        if count == 1 or cut:
            pick += [("first", int(order[first])), ("last", int(order[first + count - 1]))] if count > 1 else \
                [("single", int(order[first]))]
    pick.append(("dm", case["dms"].index(ic.DM)))
    seen, out = set(), []
    for kind, k in pick:
        if k not in seen:
            seen.add(k)
            out.append((kind, k))
    return out


@pytest.mark.parametrize("band", ["upright", "inverted"])
def test_every_trial_and_planted_alignment_against_float64(ctx, band):
    """pulses along the first and last trial of every spread-cut group, every single-trial group and the trial at dm,
    each at its own time; three calls, each raising a different kind of trial (group-first, group-last, single or dm)
    above the others so that it is the best. Every trial against float64, each planted trial's boxcar-1 peak at its
    time, and the best trial's series sample by sample."""
    case = CASES[band]
    s, sm, T = _geometry(case)
    chosen = _chosen(case)
    kinds = [k for k, _ in chosen]
    assert "first" in kinds and "last" in kinds and (band == "inverted" or "single" in kinds)
    times = {k: 200 + i * ((T - 400) // len(chosen)) for i, (_, k) in enumerate(chosen)}
    order = ["first", "last", "single" if band == "upright" else "dm"]
    for call, kind in enumerate(order):
        target = next(k for kk, k in chosen if kk == kind)
        x = _spectrum(ic.C, case["time_count"], 100 + call)
        for _, k in chosen:
            _plant(x, s, sm, k, times[k], 1.6 if k == target else 1.0)
        (res, (psnr, pidx), best, hs), v = _check_all(ctx, x, case)
        assert best == target, (kind, best, target)
        for _, k in chosen:
            assert int(pidx[k][0]) == times[k], (kind, k, int(pidx[k][0]), times[k])
        assert res[best].signal_count[0] > 0


def test_results_do_not_depend_on_trial_order(ctx):
    """each trial's series is the same fp32 sum in channel order whatever group it lands in: a shuffled list, the
    reversed list and one with duplicates give the sorted list's results permuted, byte for byte"""
    base = CASES["upright"]
    s, sm, T = _geometry(base)
    x = _spectrum(ic.C, base["time_count"], 7)
    k = base["dms"].index(ic.DM)
    _plant(x, s, sm, k, T // 2, 1.2)
    ref = _search(ctx, x, base)
    _check_all(ctx, x, base, ref)
    key = {d: i for i, d in enumerate(base["dms"])}
    for name in ("shuffled", "reversed", "duplicates"):
        case = CASES[name]
        res, (psnr, pidx), best, hs = _search(ctx, x, case)
        for j, d in enumerate(case["dms"]):
            i = key[d]
            assert bytes(memoryview(res[j])) == bytes(memoryview(ref[0][i])), (name, j)
            assert np.array_equal(psnr[j], ref[1][0][i]) and np.array_equal(pidx[j], ref[1][1][i]), (name, j)
        assert case["dms"][best] == base["dms"][ref[2]], name
        assert case["dms"].index(case["dms"][best]) == best  # the lowest index of a duplicated best
        assert np.array_equal(hs, ref[3]), name


def test_table_cache_across_lists(ctx):
    """list A, a larger list B (the tables grow), another list of A's size, then A again on one context: the last call
    is bit-identical to A on a fresh context"""
    a = CASES["tail_1"]
    b = dict(CASES["inverted"], time_count=a["time_count"], reserved=0)
    a2 = dict(a, dms=[ic._f32(d + 0.01) for d in a["dms"]])
    x = _spectrum(ic.C, a["time_count"], 9)
    s, sm, T = _geometry(a)
    _plant(x, s, sm, 5, T // 3, 1.2)
    fresh = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        want = _search(fresh, x, a)
    finally:
        fresh.close()
    for case in (a, b, a2):
        _search(ctx, x, case)
    got = _search(ctx, x, a)
    assert [bytes(memoryview(r)) for r in got[0]] == [bytes(memoryview(r)) for r in want[0]]
    assert np.array_equal(got[1][0], want[1][0]) and np.array_equal(got[1][1], want[1][1]) and got[2] == want[2]
    assert np.array_equal(got[3], want[3])
    _check_all(ctx, x, a, got)


@pytest.mark.parametrize("name", ["smem_1472", "smem_1473"])
def test_shared_memory_limit_on_a_fresh_context(name):
    """the largest group spread at 1472 (exactly 48 KiB of dynamic shared memory) and 1473 (the opt-in above it), each
    as a fresh context's first call; 1473 also after a small-spread first call"""
    case = CASES[name]
    s, sm, T = _geometry(case)
    x = _spectrum(ic.C, case["time_count"], 11)
    _plant(x, s, sm, len(case["dms"]) - 1, T - 300, 1.2)
    small = dict(case, dms=[ic.DM, ic._f32(ic.DM + 0.01)])
    for warm in ([None, small] if name == "smem_1473" else [None]):
        c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
        try:
            if warm is not None:
                _check_all(c, x, warm)
            out = _check_all(c, x, case)[0]
            assert out[2] == len(case["dms"]) - 1
        finally:
            c.close()


def test_group_of_spread_exactly_1792_against_float64(ctx):
    """a group whose spread is exactly INC_SPREAD_MAX, then the trial that would make it 1793 starting the next group:
    the library's groups are the restatement's, and every trial matches float64"""
    case = CASES["spread_1792"]
    s, sm, T = _geometry(case)
    fl, bw = ic.BANDS[case["band"]]
    order, groups, gmin, gmax, spread = ig.groups(s, case["dms"])
    g_order, g_groups, g_gspan, g_spread = srtb_b200.incoherent_groups(ic.C, fl, bw, ic.SR, ic.DM, case["dms"])
    assert [tuple(g) for g in g_groups] == groups and g_spread == spread == ig.INC_SPREAD_MAX
    assert np.array_equal(g_order, order) and np.array_equal(g_gspan[:, :, 0], gmin + sm)
    x = _spectrum(ic.C, case["time_count"], 15)
    last = int(order[groups[0][1] - 1])  # the trial that brings group 0 to 1792
    _plant(x, s, sm, last, T // 2, 1.2)
    out = _check_all(ctx, x, case)[0]
    assert out[2] == last and int(out[1][1][last][0]) == T // 2


@pytest.mark.parametrize("name", ["tail_1", "tail_255", "short"])
def test_zero_filled_last_tile(ctx, name):
    """time_reserved_count = 0 and T = 1 or 255 mod 256 (or T < 256): the last tile stages samples at and past L with
    zero fill. A pulse along the trial that reaches S+ ends on the last output sample, so its last channel sample is
    x[c][L - 1]."""
    case = CASES[name]
    s, sm, T = _geometry(case)
    k = int(np.argmax(s.max(1)))
    c_edge = int(np.argmax(s[k]))
    assert T - 1 + sm + s[k, c_edge] == case["time_count"] - 1 - case["reserved"]
    x = _spectrum(ic.C, case["time_count"], 13)
    _plant(x, s, sm, k, T - 1, 1.5)
    x[c_edge, case["time_count"] - 1 - case["reserved"], 0] += 3.0  # the sample only the last output reads
    (res, (psnr, pidx), best, hs), v = _check_all(ctx, x, case)
    assert best == k and int(pidx[k][0]) == T - 1


@pytest.mark.parametrize("label", list(ic.LONG_T))
def test_series_longer_than_65535_tiles(ctx, label):
    """C = 2, three trials, T = 65535 * 256 (the longest series one tile per CTA covers), one sample more, and 2^24 +
    2^17: every trial against float64 and a pulse on the last samples of trial 1, past tile 65535"""
    T = ic.LONG_T[label]
    fl, bw = ic.LONG_BAND
    s, sp, sm = io.shifts(ic.LONG_C, fl, bw, ic.LONG_SR, ic.DM, ic.LONG_DMS)
    L = T + sp + sm
    g = torch.Generator(device="cuda").manual_seed(17)
    x = torch.randn((ic.LONG_C, L, 2), device="cuda", generator=g, dtype=torch.float32)
    _plant(x, s, sm, 1, T - 3, 10.0)
    nb = 3  # boxcars 1, 2, 4
    hs = np.zeros((nb, T), np.float32)
    res, (psnr, pidx), best, hs = ctx.incoherent_dm_search(x, L, ic.LONG_C, 0, fl, bw, ic.LONG_SR, ic.DM, ic.LONG_DMS,
                                                           SNR, CHAN_THR, 4, hs)
    assert res[0].time_series_count == T and res[0].n_boxcars == nb
    v, zc = _truth(x, s, sm, T)
    del x
    torch.cuda.empty_cache()
    for d in range(3):
        _check_trial(res[d], psnr[d], pidx[d], v[d], zc, ic.LONG_C, (label, d), hs if d == best else None, maxbox=4)
    assert best == 1 and int(pidx[1][0]) == T - 3


def _pulse(n, t0, f_low, bw, d0, amp):
    """bench.dispersed_pulse over the whole recording (circular, negligible at the ends): a pulse dispersed at d0 whose
    top-of-band arrival is sample t0"""
    return bench.dispersed_pulse(n, {"f_low": f_low, "bw": bw, "dm": d0}, amp=amp, t0_frac=(t0 + 0.5) / n)


def test_executable_finds_a_pulse_in_the_block_overlap(tmp_path):
    """src/srtb_b200 with --incoherent_dm_list on a two-stream recording of two blocks, baseband_reserve_sample = 1,
    C = 1024 and a trial list cut by spread: a pulse whose arrival lies in the overlap that nsamps_reserved_max() adds
    for the search (block 0's unsearched tail, block 1's searched head) is found in block 1 at its trial DM, at the
    boxcar-1 index the block step N - overlap predicts. A second pulse in block 0's searched part is found there.
    The block path leaves out R / C spectrum samples (R = nsamps_reserved()), so each block searches
    T = L - R / C - S+ - S- series samples, while blocks start (N - overlap) / 2C = L - R / 2C - S+ - S- apart."""
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    C_, f_low, bw, dm, n = 1024, 1000.0, 500.0, 0.5, 1 << 24
    sr = 2e6 * bw
    dms = [ic._f32(dm - 0.45 + 0.15 * i) for i in range(17)]  # dm - 0.45 .. dm + 1.95
    s, sp, sm = io.shifts(C_, f_low, bw, sr, dm, dms)
    _, groups, _, _, spread = ig.groups(s, dms)
    assert len(groups) >= 2 and all(c < ig.INC_GROUP for _, c in groups[:-1]), groups  # cut by spread
    R = srtb_b200.nsamps_reserved(n, C_, f_low, bw, sr, dm, True)
    overlap = R + 2 * C_ * (sp + sm)
    step = n - overlap
    assert R % (2 * C_) == 0 and 0 < overlap < n
    L = n // (2 * C_)
    T = L - R // C_ - sp - sm  # each block searches series indices j < T
    S = step // (2 * C_)  # block 1's first spectrum sample
    assert step % (2 * C_) == 0 and S == L - R // (2 * C_) - sp - sm and T > 1000
    d_b, d_a = dms[6], dms[1]  # the pulses' DMs, trials of their own
    j_b = S + (sp + sm) // 2  # global series index of pulse B: in the search's share of the overlap
    j_a = T // 3
    assert T <= j_b and j_b - S < T
    total = -(-(n + step) // (1 << 19)) << 19  # two blocks and a little more; bench.dispersed_pulse takes 2^19 multiples
    t_b, t_a = 2 * C_ * (j_b + sm), 2 * C_ * (j_a + sm)  # top-of-band arrivals, at spectrum sample starts
    streams = []
    rng = np.random.default_rng(31)
    for st in range(2):
        v = rng.standard_normal(total) * 20.0
        if st == 1:
            v += _pulse(total, t_b, f_low, bw, d_b, 1500.0) + _pulse(total, t_a, f_low, bw, d_a, 1500.0)
        streams.append(np.clip(np.round(v), -127, 127).astype(np.int8))
    raw = np.empty(2 * total, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = streams[0].reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = streams[1].reshape(-1, 2)
    inp = tmp_path / "bb.bin"
    raw.tofile(inp)
    prefix = tmp_path / "cand_"
    cfg = tmp_path / "seam.cfg"
    cfg.write_text(f"""# incoherent search across a block seam
baseband_input_count = 2 ** 24
baseband_input_bits = -8
baseband_format_type = naocpsr_snap1
baseband_freq_low = {f_low}
baseband_bandwidth = {bw}
baseband_sample_rate = {sr}
baseband_reserve_sample = 1
dm = {dm}
spectrum_channel_count = {C_}
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 8
signal_detect_max_boxcar_length = 16
input_file_path = {inp}
baseband_output_file_prefix = {prefix}
log_level = 3
""")
    dm_list = ",".join(f"{d:.9g}" for d in dms)
    r = subprocess.run([str(exe), "--config_file_name", str(cfg), "--incoherent_dm_list", dm_list, "--ring_depth", "2"],
                       capture_output=True, text=True, timeout=300,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    assert f"block overlap {overlap} samples" in r.stderr, r.stderr[-3000:]
    csvs = sorted(tmp_path.glob("cand_*.1.dm_sweep.csv"), key=lambda p: int(p.name.split(".")[0][len("cand_"):]))
    # which block each file is: its .bin holds the block's bytes, block b starting at sample b * step
    blocks = []
    for p in csvs:
        stem = p.name.split(".")[0]
        b = np.fromfile(tmp_path / f"{stem}.bin", np.int8)
        starts = [i for i in range(3) if np.array_equal(b[:4096], raw[2 * i * step:2 * i * step + 4096])]
        assert len(starts) == 1, p.name
        blocks.append(starts[0])
    assert blocks[:2] == [0, 1], (blocks, [p.name for p in csvs])

    def peak(path):
        rows = [ln.split(",") for ln in path.read_text().splitlines()[1:]]
        box1 = [row for row in rows if row[2] == "1"]
        top = max(box1, key=lambda row: float(row[6]))
        return float(top[0]), int(top[7]), float(top[6])

    dm0, idx0, snr0 = peak(csvs[0])
    dm1, idx1, snr1 = peak(csvs[1])
    assert dm0 == pytest.approx(d_a) and idx0 == j_a, (dm0, idx0, snr0)
    assert dm1 == pytest.approx(d_b) and idx1 == j_b - S, (dm1, idx1, snr1, j_b, S, T)
