"""Events of the block path (srtb_b200_submit_block_events / collect_block_events) on the GPU: every stream's and the
total intensity's events against the maximal runs of the series process_block returns for the same block
(tests/candidates_oracle.runs), at one shape per detector route; several blocks in flight, a ticket wrap and one lane
against two; bit-identical headers, series and spectra against submit_block_ex with the documented launch delta;
truncated lists, counts only, detection disabled and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import srtb_b200  # noqa: E402
from candidates_oracle import runs  # noqa: E402
from test_gpu_parity import _from_device_ptr, make_block_config  # noqa: E402

MB = srtb_b200.MAX_BOXCARS
E_INVALID = -1
SNR, MAXBOX = 4.0, 256
EV_DT = srtb_b200._dtype_of(srtb_b200.Event)


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).pin_memory()


def _q(v):
    return np.clip(np.round(v), -127, 127).astype(np.int8)


def _snap1(a, b):
    raw = np.empty(2 * a.size, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = a.reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = b.reshape(-1, 2)
    return raw


def _gain(C_):
    """a burst's amplitude gain: about 6 sigma per spectrum sample in the sum over C channels. Weak enough that even in
    a row of 256 samples the bursts leave the detector's variance, and so its threshold, near the noise's"""
    return np.float32(np.sqrt(1 + 6 / np.sqrt(C_)))


def _pol(n, C_, seed, pulses, sigma=20.0):
    """one polarisation: noise plus bursts of _gain(C) times the noise's amplitude, each (start, width) in spectrum
    samples of 2C baseband samples. At dm = 0 the chirp is the identity, so each burst stays where it was put."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(n).astype(np.float32) * np.float32(sigma)
    for t0, w in pulses:
        a, b = t0 * 2 * C_, (t0 + w) * 2 * C_
        v[a:b] *= _gain(C_)
    return _q(v)


def _block(n, C_, seed, pulses):
    return _snap1(_pol(n, C_, seed, pulses), _pol(n, C_, seed + 1, pulses))


def _cfg(n, C_, sum_=1, avg_thr=5.0, chan_thr=0.9):
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, C_, 0.0, f_low=1000.0, bw=64.0, fs=128e6,
                            avg_thr=avg_thr, sk_thr=1.3, snr=SNR, chan_thr=chan_thr, maxbox=MAXBOX)
    cfg.signal_detect_sum_streams = sum_
    return cfg


def _L(cfg):
    n = cfg.baseband_input_count
    return n // 2 // min(cfg.spectrum_channel_count, n // 2)


def _truth(ctx, cfg, raw, rows):
    """process_block's headers and every series, and the runs of each detector's rows as an Event array"""
    L = _L(cfg)
    h = np.zeros((rows, MB, L), np.float32)
    res = ctx.process_block(cfg, _pinned(raw), raw.size, h, True)
    assert len(res) == rows
    out = []
    for r in range(rows):
        ev = []
        hd = res[r]
        if hd.detect_enabled:
            for b in range(hd.n_boxcars):
                for (b0, e0, pk, snr) in runs(h[r, b, :hd.series_length[b]], hd.threshold[b], hd.variance[b]):
                    ev.append((b0, e0, pk, snr, 0, b, r))
        out.append(np.array(ev, EV_DT))
    return res, h, out


def _same_events(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("begin", "end", "peak_index", "trial", "boxcar", "stream"):
        assert np.array_equal(got[f], want[f]), (what, f)
    assert got["snr"].tobytes() == want["snr"].tobytes(), what  # bit-equal


def _bytes(r):
    return bytes(memoryview(r))


def _host_rows(ptr, rows, L):
    buf = (C.c_float * (rows * MB * L)).from_address(ptr)
    return np.frombuffer(buf, np.float32).reshape(rows, MB, L).copy()


def _ring(ctx, cfg, raw, max_events=None):
    """one block through the ring: (results, positive series, spectra, events...) copied out before the next submit"""
    d = torch.from_numpy(raw.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    if max_events is None:
        t = ctx.submit_block_ex(cfg, d, raw.size, on_device=True)
        res, sp, spec = ctx.collect_block_ex(t)
        extra = None
    else:
        t = ctx.submit_block_events(cfg, d, raw.size, max_events, on_device=True)
        res, sp, spec, ev, tot, sev, stot = ctx.collect_block_events(t)
        extra = (ev, tot, sev, stot)
    launches = ctx.launch_count - n0
    L = _L(cfg)
    series = _host_rows(sp, len(res), L)
    C_ = min(cfg.spectrum_channel_count, cfg.baseband_input_count // 2)
    spectra = [_from_device_ptr(p, C_ * L) for p in spec]
    return res, series, spectra, extra, launches


# one shape per detector route (log2 n per stream, C): L = 512 (eight-point row kernel), 2048 (chirp-fused
# sixteen-point row kernel), 16384 at the config #3 geometry (sweep-order route), 2^15 (long-row path), 256 (unfused
# detect_enqueue)
ROUTES = [(20, 1024), (22, 1024), (26, 2048), (22, 64), (20, 2048)]


def _pulses(L, shift=0):
    """four bursts of widths 1 to 8 spread over the block"""
    return [((L * k) // 5 + shift, w) for k, w in zip(range(1, 5), (1, 2, 4, 8))]


@pytest.mark.parametrize("logn,C_", ROUTES, ids=lambda v: str(v))
def test_ring_events_equal_runs_of_process_block_series(ctx, logn, C_):
    n = 1 << logn
    L = n // 2 // C_
    raw = _block(n, C_, logn, _pulses(L))
    cfg = _cfg(n, C_)
    res_t, _, truth = _truth(ctx, cfg, raw, 3)
    plain = _ring(ctx, cfg, raw)
    res, series, spectra, (ev, tot, sev, stot), launches = _ring(ctx, cfg, raw, max_events=1 << 16)
    # the events equal the runs of the synchronous entry's series, for both streams and the sum
    for s in range(2):
        assert tot[s] == len(truth[s]) > 0, (s, tot[s], len(truth[s]))
        _same_events(ev[s], truth[s], f"stream {s}")
    assert stot == len(truth[2]) > 0
    _same_events(sev, truth[2], "sum")
    assert np.all(sev["stream"] == 2)
    # the lengths of a row's events add up to its signal count
    for r, e in enumerate(ev + [sev]):
        for b in range(res[r].n_boxcars):
            sel = e["boxcar"] == b
            assert int((e["end"][sel] - e["begin"][sel]).sum()) == res[r].signal_count[b]
    # everything else is bit-identical to submit_block_ex, with two launches more per stream and per sum
    p_res, p_series, p_spectra, _, p_launches = plain
    assert launches - p_launches == 2 * 3
    for r in range(3):
        assert _bytes(res[r]) == _bytes(p_res[r]) == _bytes(res_t[r]), r
        for b in range(res[r].n_boxcars):
            if res[r].signal_count[b] > 0:
                assert np.array_equal(series[r, b, :res[r].series_length[b]],
                                      p_series[r, b, :res[r].series_length[b]]), (r, b)
    for s in range(2):
        assert spectra[s].tobytes() == p_spectra[s].tobytes(), s


def test_sum_events_with_a_channel_zapped_in_one_polarisation(ctx):
    """a tone in stream 0 only: SK zaps its channel there, the sum leaves it out of both, and the sum's events still
    equal the runs of the sum's series"""
    n, C_ = 1 << 22, 256
    L = n // 2 // C_
    t = np.arange(n)
    rng = np.random.default_rng(9)
    a = rng.standard_normal(n) * 20 + 40 * np.cos(2 * np.pi * (77 + 0.5) / (2 * C_) * t)
    for t0, w in _pulses(L):
        a[t0 * 2 * C_:(t0 + w) * 2 * C_] *= _gain(C_)
    raw = _snap1(_q(a), _pol(n, C_, 10, _pulses(L)))
    cfg = _cfg(n, C_, avg_thr=1e30)  # s1 off: the tone must reach SK
    res_t, _, truth = _truth(ctx, cfg, raw, 3)
    assert res_t[0].zero_count != res_t[1].zero_count, "the tone should be zapped in one polarisation only"
    res, _, _, (ev, tot, sev, stot), _ = _ring(ctx, cfg, raw, max_events=1 << 16)
    for s in range(2):
        _same_events(ev[s], truth[s], f"stream {s}")
    assert stot == len(truth[2]) > 0
    _same_events(sev, truth[2], "sum")


def _lists_bytes(ev, sev):
    return b"".join(e.tobytes() for e in ev) + (sev.tobytes() if sev is not None else b"")


def _three_in_flight(c, cfg, raws, max_events=4096):
    ds = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in raws]
    torch.cuda.synchronize()
    tickets = [c.submit_block_events(cfg, d, r.size, max_events, on_device=True) for d, r in zip(ds, raws)]
    out = []
    for t in tickets:
        res, _, _, ev, tot, sev, stot = c.collect_block_events(t)
        out.append((res, ev, tot, sev, stot))
    return tickets, out


def test_blocks_in_flight_each_collect_its_own_list(ctx):
    n, C_ = 1 << 22, 1024
    L = n // 2 // C_
    cfg = _cfg(n, C_)
    raws = [_block(n, C_, 50 + 7 * k, _pulses(L, shift=37 * k)) for k in range(srtb_b200.RING_SLOTS)]
    truths = [_truth(ctx, cfg, r, 3)[2] for r in raws]

    def check(out):
        for k, (res, ev, tot, sev, stot) in enumerate(out):
            for s in range(2):
                _same_events(ev[s], truths[k][s], f"block {k} stream {s}")
            _same_events(sev, truths[k][2], f"block {k} sum")

    _, out = _three_in_flight(ctx, cfg, raws)
    check(out)
    # the same across a ticket wrap
    ctx.debug_set_submit_count((srtb_b200.RING_SLOTS << 28) - 2)
    tickets, out_w = _three_in_flight(ctx, cfg, raws)
    assert tickets[-1] < tickets[0], tickets
    check(out_w)
    ctx.debug_set_submit_count(0)
    # one lane and two lanes list the same bytes
    lists = []
    for lanes in ("1", "2"):
        old = os.environ.get("SRTB_B200_LANES")
        os.environ["SRTB_B200_LANES"] = lanes
        try:
            c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            if old is None:
                del os.environ["SRTB_B200_LANES"]
            else:
                os.environ["SRTB_B200_LANES"] = old
        try:
            _, o = _three_in_flight(c, cfg, raws)
            lists.append([_lists_bytes(ev, sev) for (_, ev, _, sev, _) in o])
        finally:
            c.close()
    assert lists[0] == lists[1]
    assert lists[0] == [_lists_bytes(ev, sev) for (_, ev, _, sev, _) in out]


def test_truncated_lists_counts_only_and_detection_disabled(ctx):
    n, C_ = 1 << 22, 1024
    L = n // 2 // C_
    raw = _block(n, C_, 77, _pulses(L))
    cfg = _cfg(n, C_)
    ev, tot, sev, stot = _ring(ctx, cfg, raw, max_events=1 << 16)[3]
    assert min(tot) > 3 and stot > 3
    # a small cap: the first events in list order, the true totals
    _, _, _, (ev3, tot3, sev3, stot3), _ = _ring(ctx, cfg, raw, max_events=3)
    assert tot3 == tot and stot3 == stot
    for s in range(2):
        assert ev3[s].tobytes() == ev[s][:3].tobytes()
    assert sev3.tobytes() == sev[:3].tobytes()
    # counts only
    _, _, _, (ev0, tot0, sev0, stot0), _ = _ring(ctx, cfg, raw, max_events=0)
    assert tot0 == tot and stot0 == stot and all(len(e) == 0 for e in ev0) and len(sev0) == 0
    # detection disabled (channel threshold 0): nothing is listed
    cfg_off = _cfg(n, C_, chan_thr=0.0)
    res, _, _, (evd, totd, sevd, stotd), _ = _ring(ctx, cfg_off, raw, max_events=1024)
    assert all(not r.detect_enabled for r in res)
    assert totd == [0, 0] and stotd == 0 and all(len(e) == 0 for e in evd)


def test_refusals(ctx):
    n, C_ = 1 << 20, 1024
    raw = _block(n, C_, 3, [])
    cfg = _cfg(n, C_, sum_=0)
    d = torch.from_numpy(raw.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    lib = ctx.lib
    # submit: max_events above 2^32, before any launch
    before = ctx.launch_count
    rc = lib.srtb_b200_submit_block_events(ctx.h, C.byref(cfg), d.data_ptr(), raw.size, 1,
                                           C.byref(srtb_b200.BlockOutputs()), (1 << 32) + 1)
    assert rc == E_INVALID and ctx.launch_count == before
    # collect_block_events on a plain ticket: refused, and the ticket is still there to collect
    t = ctx.submit_block_ex(cfg, d, raw.size, on_device=True)
    res = (srtb_b200.DetectResult * 5)()
    evp, n_ev = C.c_void_p(), (C.c_uint64 * 5)()
    assert lib.srtb_b200_collect_block_events(ctx.h, t, res, None, None, C.byref(evp), n_ev) == E_INVALID
    ctx.collect_block_ex(t)
    # a null n_events, a null h_events with max_events > 0; max_events == 0 takes a null h_events
    t = ctx.submit_block_events(cfg, d, raw.size, 8, on_device=True)
    assert lib.srtb_b200_collect_block_events(ctx.h, t, res, None, None, C.byref(evp), None) == E_INVALID
    assert lib.srtb_b200_collect_block_events(ctx.h, t, res, None, None, None, n_ev) == E_INVALID
    assert lib.srtb_b200_collect_block_events(ctx.h, t, res, None, None, C.byref(evp), n_ev) == 2
    ctx._event_caps.pop(t, None)
    ctx._sum_tickets.pop(t, None)
    t = ctx.submit_block_events(cfg, d, raw.size, 0, on_device=True)
    assert lib.srtb_b200_collect_block_events(ctx.h, t, res, None, None, None, n_ev) == 2
    ctx._event_caps.pop(t, None)
    ctx._sum_tickets.pop(t, None)


# ---- the executable ------------------------------------------------------------------------------------------------
import resource  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402
from pathlib import Path  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

X_N, X_C, X_FLOW, X_BW, X_DM, X_BLOCKS = 1 << 22, 256, 1000.0, 64.0, 0.5, 3
X_FS = 2 * X_BW * 1e6


def _x_geometry():
    """(R, L, L', share): reserved baseband samples, row length, samples the detector searches, a block's share"""
    R = srtb_b200.nsamps_reserved(X_N, X_C, X_FLOW, X_BW, X_FS, X_DM, True)
    L = X_N // 2 // X_C
    return R, L, L - R // X_C, (X_N - R) // (2 * X_C)


def _x_recording(streams, seed):
    """X_BLOCKS blocks' worth of 8-bit noise with pulses dispersed at X_DM: inside blocks and on both sides of the
    boundary between blocks 0 and 1, each outside the span no block searches. Returns (raw, pulse times in samples)."""
    R, L, Lp, share = _x_geometry()
    step = X_N - R
    T = (X_BLOCKS - 1) * step + X_N
    T2 = -(-T // (1 << 19)) << 19  # dispersed_pulse's length: whole chunks of its spectrum; cut back to T below
    two_c = 2 * X_C
    t0s = [int(0.3 * step), (Lp - 40) * two_c + 7, step + 25 * two_c + 3, step + int(0.55 * step),
           2 * step + int(0.4 * step)]
    w = {"f_low": X_FLOW, "bw": X_BW, "dm": X_DM}
    pulse = sum(bench.dispersed_pulse(T2, w, amp=1500.0, t0_frac=t / T2) for t in t0s)[:T]
    rng = np.random.default_rng(seed)
    pols = [_q(rng.standard_normal(T).astype(np.float32) * np.float32(20) + pulse) for _ in range(streams)]
    raw = pols[0] if streams == 1 else _snap1(pols[0], pols[1])
    return raw, t0s


def _x_run(tmp_path, name, raw, fmt, extra):
    d = tmp_path / name
    d.mkdir()
    inp = d / "bb.bin"
    raw.tofile(inp)
    cfg = d / "x.cfg"
    cfg.write_text(f"""baseband_input_count = {X_N}
baseband_input_bits = -8
baseband_format_type = {fmt}
baseband_freq_low = {X_FLOW}
baseband_bandwidth = {X_BW}
baseband_sample_rate = {X_FS}
baseband_reserve_sample = 1
dm = {X_DM}
spectrum_channel_count = {X_C}
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 8
signal_detect_max_boxcar_length = 256
input_file_path = {inp}
baseband_output_file_prefix = {d / "out_"}
log_level = 3
""")
    # no core file if the executable aborts: a CUDA process's image is large
    r = subprocess.run([str(ROOT / "src" / "srtb_b200"), "--config_file_name", str(cfg), "--ring_depth", "3"] + extra,
                       capture_output=True, text=True, timeout=600,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    inp.unlink()
    return d


def _rows(paths):
    out = []
    for p in paths:
        lines = p.read_text().splitlines()
        assert lines[0] == "snr,dm,boxcar_length,sample,time,members,dm_low,dm_high,span_begin,span_end,trial,peak_index"
        out += [dict(zip(lines[0].split(","), ln.split(","))) for ln in lines[1:]]
    return out


def _check_pulses(rows, t0s):
    """each pulse is exactly one row, at its time within one boxcar window plus one sample; no other rows"""
    two_c = 2 * X_C
    assert len(rows) == len(t0s), rows
    for t0 in t0s:
        hit = [r for r in rows if abs(float(r["time"]) * X_FS - t0) <= (int(r["boxcar_length"]) + 1) * two_c]
        assert len(hit) == 1, (t0, rows)
        r = hit[0]
        assert float(r["dm"]) == X_DM == float(r["dm_low"]) == float(r["dm_high"]) and r["trial"] == "0"


def _outputs(d):
    """the run's output files in block order, by their name after the counter"""
    return sorted((p.name.split("_", 1)[1].split(".", 1)[1], p.read_bytes()) for p in d.iterdir()
                  if p.name.startswith("out_"))


def test_share_covers_what_the_detector_searches():
    """L' = L - R/C <= the share (N - R) / 2C, so no pulse is listed by two blocks; R/(2C) samples per share are
    searched by no block"""
    R, L, Lp, share = _x_geometry()
    assert R > 0 and Lp <= share and share - Lp == (X_N - R) // (2 * X_C) - (L - R // X_C)
    print(f"R = {R}, L = {L}, L' = {Lp}, share = {share}, unsearched = {share - Lp}")


def test_detector_searches_l_prime(ctx):
    R, L, Lp, share = _x_geometry()
    cfg = make_block_config(X_N, -8, srtb_b200.FORMAT_SIMPLE, X_C, X_DM, f_low=X_FLOW, bw=X_BW, fs=X_FS)
    cfg.baseband_reserve_sample = 1
    raw = _q(np.random.default_rng(5).standard_normal(X_N) * 20)
    res = ctx.process_block(cfg, _pinned(raw), raw.size)
    assert res[0].time_series_count == Lp <= share


def test_executable_single_stream(tmp_path):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    raw, t0s = _x_recording(1, 11)
    d = _x_run(tmp_path, "on", raw, "simple", ["--signal_detect_candidates", "1"])
    _check_pulses(_rows(sorted(d.glob("out_*.0.candidates.csv"))), t0s)


def test_executable_dual_polarisation_with_sum(tmp_path):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    raw, t0s = _x_recording(2, 12)
    d = _x_run(tmp_path, "on", raw, "naocpsr_snap1",
               ["--signal_detect_candidates", "1", "--signal_detect_sum_polarizations", "1"])
    for s in range(2):
        _check_pulses(_rows(sorted(d.glob(f"out_*.{s}.candidates.csv"))), t0s)
    _check_pulses(_rows(sorted(d.glob("out_*.sum.candidates.csv"))), t0s)
    # with the key at 0, the same files as a run without it
    off = _x_run(tmp_path, "off", raw, "naocpsr_snap1", ["--signal_detect_sum_polarizations", "1"])
    zero = _x_run(tmp_path, "zero", raw, "naocpsr_snap1",
                  ["--signal_detect_candidates", "0", "--signal_detect_sum_polarizations", "1"])
    a, b = _outputs(off), _outputs(zero)
    assert a and [n for n, _ in a] == [n for n, _ in b] and a == b
    assert not any("candidates" in n for n, _ in a)
