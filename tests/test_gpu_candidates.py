"""The single-pulse event list on the device (csrc/events.cuh) and the candidates clustered from it.

series_events on crafted series (runs at tile edges, whole rows above threshold, values exactly at it, ties, skipped
trials, zero variance, truncation) against the exact numpy restatement in candidates_oracle.py; the DM searches'
_events entries against their plain entries (bit-identical results) and against their own signal counts and peaks; and
a block with two dispersed pulses and a broadband spike, which clusters into exactly three candidates."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import candidates_oracle as oracle  # noqa: E402
import incoherent_oracle as io  # noqa: E402
import srtb_b200  # noqa: E402
from test_gpu_dm_sweep_candidates import CASES, _block, _cfg, _pinned  # noqa: E402
from test_gpu_incoherent_search import _block_cfg, _pulse_block, _random_spectrum, _to_device  # noqa: E402

import bench  # noqa: E402  (test_gpu_incoherent_search put the repository root on sys.path)

SNR, CHAN_THR, MAXBOX = 6.0, 0.9, 64
FIELDS = ("begin", "end", "peak_index", "snr", "trial", "boxcar", "stream")


def _header(n_boxcars, lengths, thr, var, enabled=1):
    r = srtb_b200.DetectResult()
    r.detect_enabled = enabled
    r.n_boxcars = n_boxcars
    for b in range(n_boxcars):
        r.boxcar_length[b] = 1 << b
        r.series_length[b] = lengths[b]
        r.threshold[b] = thr[b]
        r.variance[b] = var[b]
    return r


def _oracle_events(series, results):
    """the event list of rows series[y][b][:series_length[b]] in (trial, boxcar, begin) order"""
    out = []
    for y, r in enumerate(results):
        if not r.detect_enabled:
            continue
        for b in range(r.n_boxcars):
            v = series[y][b][:r.series_length[b]]
            for (b0, e0, p, snr) in oracle.runs(v, r.threshold[b], r.variance[b]):
                out.append((b0, e0, p, snr, y, b, 0))
    return out


def _same(got, want, where=""):
    assert len(got) == len(want), (where, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        for f, v in zip(FIELDS, w):
            if f == "snr":
                assert np.float32(g[f]).tobytes() == np.float32(v).tobytes(), (where, i, g, w)
            else:
                assert int(g[f]) == int(v), (where, i, f, g, w)


def test_series_events_crafted(ctx):
    rng = np.random.default_rng(5)
    stride = (1 << 20) + 3
    nb = 3
    series = np.zeros((4, nb, stride), np.float32)
    results = []
    # trial 0: a noisy row crossing every power of two from 2^8 to 2^16, a whole row above threshold, variance 0
    n0 = (1 << 17) + 5
    v = rng.standard_normal(n0).astype(np.float32)
    v[v > 1.0] *= 0.5  # fewer runs of the noise itself
    for k in range(8, 17):
        p = 1 << k
        v[p - 3:p + 4] = np.float32(2.0) + np.arange(7, dtype=np.float32) * np.float32(0.01 * k)
    v[0:3] = 3.0  # a run starting at 0
    v[n0 - 2:] = 3.0  # one ending at n - 1
    v[5000:5010] = 1.0  # exactly at the threshold: not above
    v[7000:7006] = [2.0, 4.0, 1.5, 4.0, 4.0, 2.0]  # tied maxima: the smallest index
    series[0, 0, :n0] = v
    series[0, 1, :] = rng.uniform(1.5, 9.0, stride).astype(np.float32)  # whole row above
    series[0, 2, :1000] = np.where(np.arange(1000) % 7 == 0, 5.0, 0.0)
    results.append(_header(3, [n0, stride, 1000], [1.0, 1.0, 1.0], [4.0, 2.5, 0.0]))
    # trial 1: detection disabled, everything above: skipped
    series[1, :, :] = 10.0
    results.append(_header(2, [stride, 100], [1.0, 1.0], [1.0, 1.0], enabled=0))
    # trials 2, 3: rows of different lengths at tile edges
    for y, lens in ((2, [4096, 4097]), (3, [8191, 1])):
        for b, n in enumerate(lens):
            series[y, b, :n] = (rng.standard_normal(n) > 1.2).astype(np.float32) * 3.0
            series[y, b, n - 1] = 3.0
        results.append(_header(2, lens, [2.0, 2.0], [1.0, 3.0]))
    d = torch.from_numpy(series).cuda()
    want = _oracle_events(series, results)
    assert len(want) > 2000
    n0_launch = ctx.launch_count
    got, total = ctx.series_events(d, stride, nb * stride, results, 1 << 20)
    assert ctx.launch_count - n0_launch <= 3
    assert total == len(want)
    _same(got, want)
    # the whole row is one event; the tied run peaks at its first 4.0; the zero-variance row has snr 0
    whole = got[(got["trial"] == 0) & (got["boxcar"] == 1)]
    assert len(whole) == 1 and whole[0]["begin"] == 0 and whole[0]["end"] == stride
    tied = got[(got["trial"] == 0) & (got["boxcar"] == 0) & (got["begin"] == 7000)]
    assert len(tied) == 1 and tied[0]["peak_index"] == 7001 and tied[0]["end"] == 7006
    assert np.all(got[(got["trial"] == 0) & (got["boxcar"] == 2)]["snr"] == 0)
    assert not np.any(got["trial"] == 1)
    # the partition: every row's lengths add up to its count of samples above threshold
    for y, r in enumerate(results):
        for b in range(r.n_boxcars if r.detect_enabled else 0):
            sel = got[(got["trial"] == y) & (got["boxcar"] == b)]
            n_above = int(np.count_nonzero(series[y, b, :r.series_length[b]] > np.float32(r.threshold[b])))
            assert int((sel["end"] - sel["begin"]).sum()) == n_above, (y, b)
    again, total2 = ctx.series_events(d, stride, nb * stride, results, 1 << 20)
    assert total2 == total and again.tobytes() == got.tobytes()
    # truncation: the first max_events and the true total
    few, total3 = ctx.series_events(d, stride, nb * stride, results, 100)
    assert total3 == total and few.tobytes() == got[:100].tobytes()


def test_series_events_rejects(ctx):
    d = torch.zeros(64, device="cuda")
    n = C.c_uint64()
    ok = (srtb_b200.DetectResult * 2)(_header(1, [32], [1.0], [1.0]), _header(1, [32], [1.0], [1.0]))
    lib, h = ctx.lib, ctx.h
    before = ctx.launch_count
    assert lib.srtb_b200_series_events(h, None, 32, 32, ok, 2, None, 0, C.byref(n)) == -1
    assert lib.srtb_b200_series_events(h, d.data_ptr(), 32, 32, ok, 2, None, 0, None) == -1
    assert lib.srtb_b200_series_events(h, d.data_ptr(), 32, 32, ok, 2, None, 5, C.byref(n)) == -1
    assert lib.srtb_b200_series_events(h, d.data_ptr(), 32, 16, ok, 2, None, 0, C.byref(n)) == -1  # rows overlap
    assert ctx.launch_count == before
    assert lib.srtb_b200_series_events(h, d.data_ptr(), 32, 32, ok, 2, None, 0, C.byref(n)) == 0


def _check_search_events(res, psnr, pidx, ev, total):
    """partition, peak records and order of a search's events (one stream)"""
    assert total == len(ev)
    keys = list(zip(ev["stream"].tolist(), ev["trial"].tolist(), ev["boxcar"].tolist(), ev["begin"].tolist()))
    assert keys == sorted(keys)
    for d, r in enumerate(res):
        for b in range(r.n_boxcars if r.detect_enabled else 0):
            sel = ev[(ev["trial"] == d) & (ev["boxcar"] == b)]
            assert int((sel["end"] - sel["begin"]).sum()) == int(r.signal_count[b]), (d, b)
            if len(sel):
                top = sel[int(np.argmax(sel["snr"]))]  # first of equal maxima: smallest begin, so smallest index
                assert np.float32(top["snr"]).tobytes() == np.float32(psnr[d][b]).tobytes(), (d, b)
                assert int(top["peak_index"]) == int(pidx[d][b]), (d, b)


@pytest.mark.parametrize("n_dm", [1, 7, 300])
@pytest.mark.parametrize("band", ["normal", "inverted"])
def test_incoherent_events(ctx, band, n_dm):
    C_, L, sr, dm = 64, 4096, 1e8, 10.0
    f_low, bw = (1000.0, 500.0) if band == "normal" else (1500.0, -500.0)
    dms = [dm + 0.25] if n_dm == 1 else list(dm + np.linspace(-0.4, 0.4, n_dm))
    if n_dm > 1:
        np.random.default_rng(n_dm).shuffle(dms)
    x = _random_spectrum(C_, L, seed=n_dm)
    s, sp, sm = io.shifts(C_, f_low, bw, sr, dm, dms)
    kp = n_dm // 3
    for c in range(C_):
        if c not in (3, 17, 40):
            x[c, 700 + sm + s[kp, c]] += 12.0
    d_x = _to_device(x)
    args = (d_x, L, C_, 100, f_low, bw, sr, dm, dms, SNR, CHAN_THR, MAXBOX)
    n0 = ctx.launch_count
    res0, (ps0, pi0), best0, hs0 = ctx.incoherent_dm_search(*args)
    n1 = ctx.launch_count
    res, (psnr, pidx), best, hs, ev, total = ctx.incoherent_dm_search_events(*args, max_events=1 << 18)
    n2 = ctx.launch_count
    assert n2 - n1 <= (n1 - n0) + 3
    assert best == best0
    assert [bytes(memoryview(r)) for r in res] == [bytes(memoryview(r)) for r in res0]
    assert ps0.tobytes() == psnr.tobytes() and pi0.tobytes() == pidx.tobytes()
    assert hs.tobytes() == hs0.tobytes()
    _check_search_events(res, psnr, pidx, ev, total)
    # the best trial's events are the runs of its returned series
    r = res[best]
    for b in range(r.n_boxcars):
        if r.signal_count[b] == 0:
            continue
        want = [(b0, e0, p, snr, best, b, 0) for (b0, e0, p, snr) in
                oracle.runs(hs[b, :r.series_length[b]], r.threshold[b], r.variance[b])]
        _same(ev[(ev["trial"] == best) & (ev["boxcar"] == b)], want, (band, n_dm, b))
    again = ctx.incoherent_dm_search_events(*args, max_events=1 << 18)
    assert again[4].tobytes() == ev.tobytes()


def test_incoherent_events_dispersed_pulse(ctx):
    n, C_, f_low, bw, dm_true, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0, 0.5
    dm = dm_true - d0
    cfg = _block_cfg(n, C_, f_low, bw, dm)
    raw = _pulse_block(n, 11, f_low, bw, dm_true)
    L = n // 2 // C_
    blk = ctx.process_block(cfg, _pinned(raw), n, np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32), True)[0]
    ptr = ctx.block_spectrum_ptr(0)
    dms = [float(np.float32(dm) + np.float32(0.05 * i)) for i in range(21)]
    args = (ptr, L, C_, L - blk.time_series_count, f_low, bw, cfg.baseband_sample_rate, dm, dms, SNR, 0.9, 256)
    res0, (ps0, pi0), best0, hs0 = ctx.incoherent_dm_search(*args)
    res, (psnr, pidx), best, hs, ev, total = ctx.incoherent_dm_search_events(*args, max_events=1 << 18)
    assert best == best0 and ps0.tobytes() == psnr.tobytes() and hs.tobytes() == hs0.tobytes()
    _check_search_events(res, psnr, pidx, ev, total)
    cands, n_c = srtb_b200.cluster_events(ev, dms)
    assert n_c >= 1
    top = cands[int(np.argmax(cands["snr"]))]
    assert abs(float(top["dm"]) - dm_true) <= 0.05 + 1e-4


def test_sweep_events_two_streams(ctx):
    case = CASES["row16_4096"]
    _, n, C_, _, _, dm = case
    cfg = _cfg(case, "naocpsr_snap1")
    raw = _block(case, "naocpsr_snap1", seed=41)
    pinned = _pinned(raw)
    dms = [0.0, 0.5 * dm, dm, 1.5 * dm]
    n0 = ctx.launch_count
    res0, (ps0, pi0), best0, hs0, sp0 = ctx.process_block_dm_sweep(cfg, pinned, raw.size, dms, outputs=True)
    n1 = ctx.launch_count
    res, (psnr, pidx), best, hs, sp, events, totals = ctx.process_block_dm_sweep_events(cfg, pinned, raw.size, dms,
                                                                                        1 << 18)
    n2 = ctx.launch_count
    streams = len(res[0])
    assert streams == 2
    assert n2 - n1 <= (n1 - n0) + 2 * len(dms) * streams
    assert best == best0 and ps0.tobytes() == psnr.tobytes() and pi0.tobytes() == pidx.tobytes()
    assert hs.tobytes() == hs0.tobytes() if hasattr(hs, "tobytes") else torch.equal(hs, hs0)
    for a, b in zip(sp, sp0):  # the dynamic spectra [C][L]: the last two floats of the buffers are not written
        assert torch.equal(a[:n], b[:n])
    for j in range(len(dms)):
        for s in range(streams):
            assert bytes(memoryview(res[j][s])) == bytes(memoryview(res0[j][s]))
    for s in range(streams):
        ev = events[s]
        assert np.all(ev["stream"] == s)
        _check_search_events([res[j][s] for j in range(len(dms))], psnr[:, s], pidx[:, s], ev, totals[s])
    assert totals[0] > 0  # stream 0 carries the pulse
    again = ctx.process_block_dm_sweep_events(cfg, pinned, raw.size, dms, 1 << 18)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(again[5], events))


def test_two_pulses_and_a_spike_are_three_candidates(ctx):
    """pulses at DM 3 and 7 at 0.25 n and 0.55 n, an undispersed broadband spike (a burst of white noise, which the 8-bit
    quantisation does not clip) at 0.8 n; the coherent sweep over DM 0 .. 10 in steps of 0.5 lists three candidates:
    each pulse within a step of its DM, the spike at DM 0, each at its time"""
    n, C_, f_low, bw = 1 << 22, 256, 1000.0, 64.0
    case = ("physics", n, C_, f_low, bw, 0.0)
    cfg = _cfg(case)
    rng = np.random.default_rng(17)
    v = rng.standard_normal(n) * 20.0
    w = {"f_low": f_low, "bw": bw}
    injected = [(3.0, 0.25), (7.0, 0.55), (0.0, 0.8)]
    for dm, t0 in injected[:2]:
        v += bench.dispersed_pulse(n, dict(w, dm=dm), amp=1000.0, t0_frac=t0)
    t_spike = int(n * injected[2][1])
    v[t_spike:t_spike + 1024] += rng.standard_normal(1024) * 40.0
    raw = np.clip(np.round(v), -127, 127).astype(np.int8)
    dms = [0.5 * i for i in range(21)]
    res, peaks, best, hs, sp, events, totals = ctx.process_block_dm_sweep_events(cfg, _pinned(raw), n, dms, 1 << 18)
    assert totals[0] == len(events[0])
    cands, n_c = srtb_b200.cluster_events(events[0], dms)
    assert n_c == 3, cands
    two_c = 2 * C_
    for c, (dm, t0) in zip(cands, injected):  # ordered by time
        assert abs(float(c["dm"]) - dm) <= 0.5 + 1e-6, (c, dm)
        sample = int(n * t0) // two_c
        assert abs(int(c["window"]) - sample) <= int(c["boxcar_length"]) + 2, (c, sample)
    assert cands[2]["trial"] == 0


def _run_exe(tmp_path, name, args):
    import resource
    import subprocess
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    subprocess.run(["make", "-C", str(root / "src")], check=True, capture_output=True)
    out = tmp_path / name
    out.mkdir()
    cfg = tmp_path / "run.cfg"
    r = subprocess.run([str(root / "src" / "srtb_b200"), "--config_file_name", str(cfg),
                        "--baseband_output_file_prefix", str(out / "c_")] + args,
                       capture_output=True, text=True, timeout=600,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _ranked_files(d):
    """{(block rank, rest of the name): bytes}: file names carry a wall-clock counter"""
    files = sorted(d.iterdir())
    counters = sorted({int(p.name[2:].split(".")[0]) for p in files if p.name[2:].split(".")[0].isdigit()})
    out = {}
    for p in files:
        head = p.name[2:].split(".")[0]
        if head.isdigit():
            out[(counters.index(int(head)), p.name[2 + len(head):])] = p.read_bytes()
        else:
            out[(-1, p.name)] = p.read_bytes()
    return out


def test_executable_candidates(tmp_path):
    """a recording of four blocks with a pulse in the coherent sweep's overlap of blocks 0 and 1 and one inside block 1:
    with --dm_search_candidates 1 each pulse is one row of all candidates.csv files, at its absolute time, for the
    coherent sweep and for the incoherent search; with the key at 0 the files are those of a run without it"""
    N, C_, f_low, bw, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0
    fs = 2 * bw * 1e6
    dm_list = "0:10:2.5"
    # the reader rewinds by the largest overlap over the trials (baseband_reserve_sample = 1)
    R = max(srtb_b200.nsamps_reserved(N, C_, f_low, bw, fs, d, True) for d in (0.0, 2.5, 5.0, 7.5, 10.0))
    step = N - R
    assert 0 < R < N // 2
    total = 3 * N
    t_pulses = [N - R // 3, step + N // 2]  # in block 0's overlap with block 1; inside block 1 only
    rng = np.random.default_rng(90)
    v = rng.standard_normal(total) * 20.0
    for t in t_pulses:
        v += bench.dispersed_pulse(total, {"f_low": f_low, "bw": bw, "dm": d0}, amp=1000.0, t0_frac=(t + 0.5) / total)
    raw = np.clip(np.round(v), -127, 127).astype(np.int8)
    inp = tmp_path / "bb.bin"
    raw.tofile(inp)
    (tmp_path / "run.cfg").write_text(f"""baseband_input_count = 2 ** 22
baseband_input_bits = -8
baseband_format_type = simple
baseband_freq_low = {f_low}
baseband_bandwidth = {bw}
baseband_sample_rate = 2 * {bw} * 1e6
baseband_reserve_sample = 1
spectrum_channel_count = {C_}
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 8
signal_detect_max_boxcar_length = 256
input_file_path = {inp}
log_level = 3
""")

    def rows_of(d):
        rows = []
        for p in sorted(d.glob("c_*.0.candidates.csv")):
            lines = p.read_text().splitlines()
            assert lines[0] == ("snr,dm,boxcar_length,sample,time,members,dm_low,dm_high,span_begin,span_end,trial,"
                                "peak_index")
            rows += [dict(zip(lines[0].split(","), ln.split(","))) for ln in lines[1:]]
        return rows

    for name, args in [("sweep", ["--dm", "0", "--dm_list", dm_list]),
                       ("incoherent", ["--dm", "4.5", "--incoherent_dm_list", "4:6:0.25"])]:
        d = _run_exe(tmp_path, name, args + ["--dm_search_candidates", "1"])
        rows = rows_of(d)
        assert len(list(d.glob("c_*.0.candidates.csv"))) >= 1
        assert len(rows) == len(t_pulses), (name, rows)
        for t, row in zip(t_pulses, sorted(rows, key=lambda r: float(r["time"]))):
            width = int(row["boxcar_length"]) * 2 * C_ / fs
            assert abs(float(row["time"]) - t / fs) <= width + 2 * C_ / fs, (name, t / fs, row)
            assert abs(float(row["dm"]) - d0) <= 2.5, (name, row)
    off = _run_exe(tmp_path, "off", ["--dm", "0", "--dm_list", dm_list, "--dm_search_candidates", "0"])
    plain = _run_exe(tmp_path, "plain", ["--dm", "0", "--dm_list", dm_list])
    a, b = _ranked_files(off), _ranked_files(plain)
    assert sorted(a) == sorted(b)
    for k in a:
        if not k[1].endswith(".check"):
            assert a[k] == b[k], k
