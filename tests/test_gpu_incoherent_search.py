"""The semi-coherent DM search (srtb_b200_incoherent_dm_search, Context.incoherent_dm_search) on the GPU: random
spectra against the float64 oracle (tests/incoherent_oracle.py) for both band orientations and 1, 7 and 300 trials, the
single trial at dm against the block path's own header, a dispersed baseband pulse found at its DM, launch counts,
determinism, argument checks, a two-stream block and the executable's --incoherent_dm_list."""
import ctypes as C
import resource
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import incoherent_oracle as io  # noqa: E402
import srtb_b200  # noqa: E402
from test_gpu_parity import _from_device_ptr, make_block_config  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

E_INVALID, E_SIZE = -1, -2
SNR, CHAN_THR, MAXBOX = 6.0, 0.9, 64


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


def _check_trial(got, peak_snr, peak_idx, want, where):
    """one trial's header and peaks against the oracle, to the tolerances float32 leaves"""
    assert got.zero_count == want["zero_count"], where
    assert bool(got.detect_enabled) == want["detect_enabled"], where
    assert got.n_boxcars == want["n_boxcars"], where
    assert got.time_series_count == want["time_series_count"], where
    for b in range(got.n_boxcars):
        assert got.boxcar_length[b] == want["boxcar_length"][b], (where, b)
        assert got.series_length[b] == want["series_length"][b], (where, b)
        assert _rel(got.variance[b], want["variance"][b]) < 1e-5, (where, b, got.variance[b], want["variance"][b])
        assert _rel(got.threshold[b], want["threshold"][b]) < 1e-5, (where, b)
        sb, thr = want["series"][b], want["threshold"][b]
        near = int(np.count_nonzero(np.abs(sb - thr) <= 1e-4 * max(abs(thr), 1e-30)))
        assert abs(int(got.signal_count[b]) - want["signal_count"][b]) <= near, (where, b)
        if peak_snr is not None:
            assert _rel(peak_snr[b], want["peak_snr"][b]) < 1e-4, (where, b, peak_snr[b], want["peak_snr"][b])
            top = np.sort(sb)[-2:] if len(sb) > 1 else sb
            tie = len(sb) > 1 and (top[1] - top[0]) <= 1e-4 * max(abs(top[1]), 1e-30)
            if not tie:
                assert int(peak_idx[b]) == want["peak_index"][b], (where, b)


def _random_spectrum(C_, L, seed, zero_channels=(3, 17, 40)):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    for c in zero_channels:
        if c < C_:
            x[c] = 0
    return x


def _to_device(x):
    return torch.from_numpy(np.ascontiguousarray(x).view(np.float32)).cuda()


@pytest.mark.parametrize("n_dm", [1, 7, 300])
@pytest.mark.parametrize("band", ["normal", "inverted"])
def test_random_spectrum_against_oracle(ctx, band, n_dm):
    C_, L, sr, dm = 64, 4096, 1e8, 10.0
    f_low, bw = (1000.0, 500.0) if band == "normal" else (1500.0, -500.0)
    if n_dm == 1:
        dms = [dm + 0.25]
    else:
        dms = list(dm + np.linspace(-0.4, 0.4, n_dm))
        np.random.default_rng(n_dm).shuffle(dms)  # any order
    x = _random_spectrum(C_, L, seed=n_dm)
    s, sp, sm = io.shifts(C_, f_low, bw, sr, dm, dms)
    kp = n_dm // 3  # a pulse along trial kp's curve
    for c in range(C_):
        if c not in (3, 17, 40):
            x[c, 700 + sm + s[kp, c]] += 12.0
    reserved = 100
    d_x = _to_device(x)
    res, (psnr, pidx), best, h_series = ctx.incoherent_dm_search(d_x, L, C_, reserved, f_low, bw, sr, dm, dms, SNR,
                                                                 CHAN_THR, MAXBOX)
    trials, want_best, _ = io.search(x, reserved, f_low, bw, sr, dm, dms, SNR, CHAN_THR, MAXBOX)
    T = L - reserved - sp - sm
    assert res[0].time_series_count == T
    for d in range(n_dm):
        _check_trial(res[d], psnr[d], pidx[d], trials[d], (band, n_dm, d))
    assert best == want_best == kp
    w = trials[best]
    assert any(c > 0 for c in w["signal_count"])
    for b in range(w["n_boxcars"]):
        if res[best].signal_count[b] > 0:
            n = w["series_length"][b]
            err = np.max(np.abs(h_series[b, :n] - w["series"][b])) / np.max(np.abs(w["series"][b]))
            assert err < 1e-4, (b, err)


def _block_cfg(n, C_, f_low, bw, dm, fmt=srtb_b200.FORMAT_SIMPLE):
    return make_block_config(n, -8, fmt, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw), avg_thr=5.0, sk_thr=1.3,
                             snr=SNR, maxbox=256)


def _pulse_block(n, seed, f_low, bw, dm, amp=1000.0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(n) * 20.0 + bench.dispersed_pulse(n, {"f_low": f_low, "bw": bw, "dm": dm}, amp=amp)
    return np.clip(np.round(v), -127, 127).astype(np.int8)


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).pin_memory()


def test_single_trial_at_dm_is_the_block_path(ctx):
    """one trial at DM = dm: every shift is 0, v is the block's column sum, and the header is the block's"""
    n, C_, f_low, bw, dm = 1 << 22, 256, 1000.0, 64.0, 5.0
    cfg = _block_cfg(n, C_, f_low, bw, dm)
    raw = _pulse_block(n, 3, f_low, bw, dm)
    L = n // 2 // C_
    h = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
    blk = ctx.process_block(cfg, _pinned(raw), n, h, True)[0]
    ptr = ctx.block_spectrum_ptr(0)
    res, (psnr, pidx), best, hs = ctx.incoherent_dm_search(ptr, L, C_, L - blk.time_series_count, f_low, bw,
                                                           cfg.baseband_sample_rate, dm, [dm], SNR, 0.9, 256)
    r = res[0]
    assert best == 0
    for f in ("zero_count", "detect_enabled", "n_boxcars", "time_series_count"):
        assert getattr(r, f) == getattr(blk, f), f
    for b in range(r.n_boxcars):
        assert r.boxcar_length[b] == blk.boxcar_length[b] and r.series_length[b] == blk.series_length[b]
        assert _rel(r.variance[b], blk.variance[b]) < 1e-5 and _rel(r.threshold[b], blk.threshold[b]) < 1e-5, b
        assert abs(int(r.signal_count[b]) - int(blk.signal_count[b])) <= 1, b
    assert sum(blk.signal_count[b] for b in range(blk.n_boxcars)) > 0
    # the best trial's positive series are the block's (same definition, another summation order)
    for b in range(r.n_boxcars):
        if r.signal_count[b] > 0 and blk.signal_count[b] > 0:
            m = r.series_length[b]
            assert np.max(np.abs(hs[b, :m] - h[b, :m])) <= 1e-4 * np.max(np.abs(h[b, :m])), b


def test_dispersed_pulse_found_at_its_dm(ctx):
    """coherent at DM_true - d0, trials dm + delta for delta in [0, 2 d0]: the best trial is DM_true, it beats delta = 0,
    and its peak index is the oracle's (pins the sign of the shifts)"""
    n, C_, f_low, bw, dm_true, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0, 0.5
    dm = dm_true - d0
    cfg = _block_cfg(n, C_, f_low, bw, dm)
    raw = _pulse_block(n, 11, f_low, bw, dm_true)
    L = n // 2 // C_
    blk = ctx.process_block(cfg, _pinned(raw), n, np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32), True)[0]
    ptr = ctx.block_spectrum_ptr(0)
    deltas = [0.05 * i for i in range(21)]
    dms = [np.float32(dm) + np.float32(dl) for dl in deltas]
    reserved = L - blk.time_series_count
    res, (psnr, pidx), best, _ = ctx.incoherent_dm_search(ptr, L, C_, reserved, f_low, bw, cfg.baseband_sample_rate,
                                                          dm, dms, SNR, 0.9, 256)
    near = int(np.argmin([abs(float(d) - dm_true) for d in dms]))
    assert best == near, (best, near, [float(psnr[d].max()) for d in range(len(dms))])
    assert psnr[best].max() > psnr[0].max()
    x = _from_device_ptr(ptr, C_ * L).reshape(C_, L)
    trials, want_best, _ = io.search(x, reserved, f_low, bw, cfg.baseband_sample_rate, dm, dms, SNR, 0.9, 256)
    assert want_best == best
    _check_trial(res[best], psnr[best], pidx[best], trials[best], "best")


def test_launch_count_does_not_grow_with_trials(ctx):
    C_, L, dm = 64, 4096, 10.0
    d_x = _to_device(_random_spectrum(C_, L, 5))
    counts = []
    for n_dm in (1, 300):
        dms = list(dm + np.linspace(-0.2, 0.2, n_dm))
        n0 = ctx.launch_count
        ctx.incoherent_dm_search(d_x, L, C_, 0, 1000.0, 500.0, 1e8, dm, dms, SNR, CHAN_THR, MAXBOX)
        counts.append(ctx.launch_count - n0)
    assert counts[0] == counts[1] <= 4, counts


def test_two_calls_are_bit_identical(ctx):
    C_, L, dm = 64, 4096, 10.0
    x = _random_spectrum(C_, L, 6)
    x[:, 1000] += 8.0
    d_x = _to_device(x)
    dms = list(dm + np.linspace(-0.3, 0.3, 77))
    a = ctx.incoherent_dm_search(d_x, L, C_, 0, 1000.0, 500.0, 1e8, dm, dms, SNR, CHAN_THR, MAXBOX)
    b = ctx.incoherent_dm_search(d_x, L, C_, 0, 1000.0, 500.0, 1e8, dm, dms, SNR, CHAN_THR, MAXBOX)
    assert [bytes(memoryview(r)) for r in a[0]] == [bytes(memoryview(r)) for r in b[0]]
    assert np.array_equal(a[1][0], b[1][0]) and np.array_equal(a[1][1], b[1][1]) and a[2] == b[2]
    assert np.array_equal(a[3], b[3])


def test_rejected_arguments_launch_nothing(ctx):
    C_, L, dm = 64, 4096, 10.0
    d_x = _to_device(_random_spectrum(C_, L, 7))
    lib = ctx.lib

    def call(ptr=None, tc=L, cc=C_, reserved=0, dms=(10.1,), n_dm=None, results=True):
        arr = (C.c_float * max(1, len(dms)))(*[float(d) for d in dms])
        res = (srtb_b200.DetectResult * max(1, len(dms)))()
        return lib.srtb_b200_incoherent_dm_search(ctx.h, d_x.data_ptr() if ptr is None else ptr, tc, cc, reserved,
                                                  1000.0, 500.0, 1e8, dm, arr, len(dms) if n_dm is None else n_dm,
                                                  SNR, CHAN_THR, MAXBOX, res if results else None, None, None, None)

    n0 = ctx.launch_count
    assert lib.srtb_b200_incoherent_dm_search(ctx.h, None, L, C_, 0, 1000.0, 500.0, 1e8, dm, None, 1, SNR, CHAN_THR,
                                              MAXBOX, None, None, None, None) == E_INVALID
    assert call(ptr=0) == E_INVALID
    assert call(results=False) == E_INVALID
    assert call(n_dm=0) == E_INVALID
    assert call(ptr=d_x.data_ptr() + 4) == E_INVALID
    assert call(reserved=L) == E_SIZE
    assert call(reserved=L + 5) == E_SIZE
    assert call(dms=(dm + 5.0,)) == E_SIZE  # shifts of ~9000 samples: T < 2
    assert call(dms=[dm] * (srtb_b200.INCOHERENT_MAX_DMS + 1)) == E_SIZE
    assert ctx.launch_count == n0
    assert call() == 0 and ctx.launch_count > n0


def test_two_stream_block(ctx):
    """naocpsr_snap1: each stream's spectrum searched on its own, against the oracle"""
    n, C_, f_low, bw, dm = 1 << 20, 64, 1000.0, 64.0, 2.0
    cfg = _block_cfg(n, C_, f_low, bw, dm, fmt=srtb_b200.FORMAT_NAOCPSR_SNAP1)
    a = _pulse_block(n, 21, f_low, bw, dm + 0.2)
    b = np.clip(np.round(np.random.default_rng(22).standard_normal(n) * 20), -127, 127).astype(np.int8)
    raw = np.empty(2 * n, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = a.reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = b.reshape(-1, 2)
    L = n // 2 // C_
    blks = ctx.process_block(cfg, _pinned(raw), raw.size, np.zeros((2, srtb_b200.MAX_BOXCARS, L), np.float32), True)
    assert len(blks) == 2
    dms = [dm + 0.05 * i for i in range(9)]
    for s in range(2):
        ptr = ctx.block_spectrum_ptr(s)
        x = _from_device_ptr(ptr, C_ * L).reshape(C_, L)
        reserved = L - blks[s].time_series_count
        res, (psnr, pidx), best, _ = ctx.incoherent_dm_search(ptr, L, C_, reserved, f_low, bw,
                                                              cfg.baseband_sample_rate, dm, dms, SNR, 0.9, 256)
        trials, want_best, _ = io.search(x, reserved, f_low, bw, cfg.baseband_sample_rate, dm, dms, SNR, 0.9, 256)
        for d in range(len(dms)):
            _check_trial(res[d], psnr[d], pidx[d], trials[d], (s, d))
        if s == 0:  # the pulse's stream; the noise stream's trials may tie within rounding
            assert best == want_best == 4


def test_executable_incoherent_dm_list(tmp_path):
    """src/srtb_b200 with --incoherent_dm_list on a file holding a pulse at d0 in stream 1, coherent at dm = d0 - 0.5:
    the S/N-versus-DM table of that stream peaks at d0 and its .tim files name d0"""
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    n, C_, f_low, bw, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0
    rng = np.random.default_rng(70)
    noise = np.clip(np.round(rng.standard_normal(n) * 20), -127, 127).astype(np.int8)
    pulse = _pulse_block(n, 71, f_low, bw, d0)
    raw = np.empty(2 * n, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = noise.reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = pulse.reshape(-1, 2)
    inp = tmp_path / "bb.bin"
    raw.tofile(inp)
    prefix = tmp_path / "cand_"
    cfg = tmp_path / "incoherent.cfg"
    cfg.write_text(f"""# semi-coherent DM search
baseband_input_count = 2 ** 22
baseband_input_bits = -8
baseband_format_type = naocpsr_snap1
baseband_freq_low = {f_low}
baseband_bandwidth = {bw}
baseband_sample_rate = 2 * {bw} * 1e6
baseband_reserve_sample = 0
dm = 4.5
spectrum_channel_count = {C_}
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 8
signal_detect_max_boxcar_length = 256
input_file_path = {inp}
baseband_output_file_prefix = {prefix}
log_level = 3
""")
    r = subprocess.run([str(exe), "--config_file_name", str(cfg), "--incoherent_dm_list", "4:6:0.25", "--ring_depth",
                        "2"], capture_output=True, text=True, timeout=300,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    assert "9 incoherent trial DM(s)" in r.stderr, r.stderr[-3000:]
    csvs = sorted(tmp_path.glob("cand_*.1.dm_sweep.csv"))
    assert len(csvs) == 1, sorted(p.name for p in tmp_path.iterdir())
    rows = [ln.split(",") for ln in csvs[0].read_text().splitlines()[1:]]
    assert sorted({float(row[0]) for row in rows}) == [4 + 0.25 * i for i in range(9)]
    best = max(rows, key=lambda row: float(row[6]))
    assert float(best[0]) == d0
    stem = csvs[0].name.split(".")[0]
    tims = sorted(tmp_path.glob(f"{stem}.dm*.tim"))
    assert tims and all(p.name.startswith(f"{stem}.dm5.") for p in tims), [p.name for p in tims]
