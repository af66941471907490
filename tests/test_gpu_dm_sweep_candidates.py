"""The DM search's candidate outputs (srtb_b200_process_block_dm_sweep_ex, Context.process_block_dm_sweep(outputs=True),
dm_sweep_chain_pipe and the executable's dm_list): per-trial peaks against the series process_block writes, the best
trial of a dispersed pulse, the best trial's re-run against the block path, negatives, argument checks, and the
executable end to end.

Where the sweep and the block path launch the same kernels (test_gpu_chirp_routes.py: chirp_variant of both paths
equal), series, spectra and headers must agree bit for bit; elsewhere within the bounds test_sweep_matches_block_path
uses."""
import ctypes as C
import resource
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import srtb_b200  # noqa: E402
from test_chirp_newton import GPU_CASES, chirp_variant  # noqa: E402
from test_gpu_parity import _from_device_ptr, make_block_config, rel_l2  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

CASES = {c[0]: c for c in GPU_CASES}
E_INVALID = -1
# rows of 512, 2^12, 2^14 and 2^16
ROW_CASES = ["unfused_512", "row16_4096", "bigrow_v3_16384", "long_n2_65536"]


def _cfg(case, fmt="simple", **kw):
    _, n, C_, f_low, bw, dm = case
    args = dict(f_low=f_low, bw=bw, fs=2e6 * abs(bw), avg_thr=5.0, sk_thr=1.3, snr=6.0, maxbox=256)
    args.update(kw)
    return make_block_config(n, -8, srtb_b200.FORMAT_BY_NAME[fmt], C_, dm, **args)


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).pin_memory()


def _snap1(a, b):
    raw = np.empty(2 * a.size, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = a.reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = b.reshape(-1, 2)
    return raw


def _noise(n, seed, sigma=20.0):
    rng = np.random.default_rng(seed)
    return np.clip(np.round(rng.standard_normal(n) * sigma), -127, 127).astype(np.int8)


def _with_pulse(n, seed, f_low, bw, dm, amp=1000.0):
    """8-bit noise (sigma 20) plus bench.dispersed_pulse: dedispersion at `dm` folds it into one impulse at 0.37 n"""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(n) * 20.0 + bench.dispersed_pulse(n, {"f_low": f_low, "bw": bw, "dm": dm}, amp=amp)
    return np.clip(np.round(v), -127, 127).astype(np.int8)


def _block(case, fmt, seed):
    _, n, _, f_low, bw, dm = case
    a = _with_pulse(n, seed, f_low, bw, dm)
    return _snap1(a, _noise(n, seed + 1)) if fmt == "naocpsr_snap1" else a


def _header_bytes(r):
    return bytes(memoryview(r))


def _exact(case):
    _, n, C_, f_low, bw, dm = case
    return chirp_variant(n, C_, f_low, bw, dm, "block") == chirp_variant(n, C_, f_low, bw, dm, "sweep")


def _sweep_ex(ctx, cfg, pinned, nbytes, dms, outputs=None):
    arr = (C.c_float * len(dms))(*[float(d) for d in dms])
    res = (srtb_b200.DetectResult * (4 * len(dms)))()
    rc = ctx.lib.srtb_b200_process_block_dm_sweep_ex(ctx.h, C.byref(cfg), srtb_b200._ptr(pinned), nbytes, 0, arr,
                                                     len(dms), res, outputs)
    return rc, res


@pytest.mark.parametrize("fmt", ["simple", "naocpsr_snap1"])
@pytest.mark.parametrize("name", ROW_CASES)
def test_ex_without_outputs_is_the_old_entry(ctx, name, fmt):
    """_ex with outputs = NULL: the old entry's headers bit for bit, and the same number of launches"""
    case = CASES[name]
    dm = case[5]
    cfg = _cfg(case, fmt)
    raw = _block(case, fmt, seed=40)
    pinned = _pinned(raw)
    dms = [0.0, 0.5 * dm, dm]
    n0 = ctx.launch_count
    old = ctx.process_block_dm_sweep(cfg, pinned, raw.size, dms)
    n1 = ctx.launch_count
    rc, res = _sweep_ex(ctx, cfg, pinned, raw.size, dms, None)
    n2 = ctx.launch_count
    streams = len(old[0])
    assert rc == streams
    assert n2 - n1 == n1 - n0
    for j in range(len(dms)):
        for s in range(streams):
            assert _header_bytes(res[j * streams + s]) == _header_bytes(old[j][s]), (j, s)


@pytest.mark.parametrize("name", ROW_CASES + ["row16_2048_inverted", "long_n0_131072_inverted"])
def test_peaks_against_block_series(ctx, name):
    """every trial's snr[b] = max(series) / sqrt(variance[b]) and peak_index[b] = first index of the maximum, with the
    series process_block writes at that DM (copy_all); exact on routes where both paths launch the same kernels"""
    case = CASES[name]
    _, n, C_, _, _, dm = case
    L = n // 2 // C_
    cfg = _cfg(case)
    raw = _block(case, "simple", seed=41)
    pinned = _pinned(raw)
    dms = [0.0, 0.5 * dm, dm]
    res, (snr, idx), best, _, _ = ctx.process_block_dm_sweep(cfg, pinned, raw.size, dms, outputs=True)
    exact = _exact(case)
    h_series = np.zeros((1, srtb_b200.MAX_BOXCARS, L), np.float32)
    for j, d in enumerate(dms):
        cfg.dm = d
        block = ctx.process_block(cfg, pinned, raw.size, h_series, True)[0]
        r = res[j][0]
        assert r.detect_enabled == block.detect_enabled and r.n_boxcars == block.n_boxcars
        for b in range(r.n_boxcars):
            v = h_series[0, b, :int(block.series_length[b])].astype(np.float64)
            var = float(np.float32(r.variance[b]))
            want = v.max() / np.sqrt(var) if var > 0 else 0.0
            if exact:
                assert int(idx[j, 0, b]) == int(np.argmax(v)), (d, b)
                assert snr[j, 0, b] == pytest.approx(want, rel=1e-6), (d, b)
            else:
                assert snr[j, 0, b] == pytest.approx(want, rel=1e-4), (d, b)
        assert np.all(snr[j, 0, r.n_boxcars:] == 0)
    assert best[0] == 2, "the pulse is dispersed at the case's DM"


def test_pulse_at_known_dm(ctx):
    """a dispersed pulse at d0 in stream 1 of a naocpsr_snap1 block, noise in stream 0: stream 1's best trial is d0's,
    positive, with its peak within one boxcar of the injected time; stream 0 stays negative"""
    n, C_, f_low, bw, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0
    L = n // 2 // C_
    raw = _snap1(_noise(n, 50), _with_pulse(n, 51, f_low, bw, d0))
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, C_, 0.0, f_low=f_low, bw=bw, fs=2e6 * bw,
                            avg_thr=5.0, sk_thr=1.3, snr=8.0, maxbox=256)
    dms = [0.0, 2.5, 5.0, 7.5, 10.0]
    res, (snr, idx), best, h_series, _ = ctx.process_block_dm_sweep(cfg, _pinned(raw), raw.size, dms, outputs=True)
    assert dms[best[1]] == d0
    r = res[best[1]][1]
    assert sum(int(c) for c in r.signal_count[:r.n_boxcars]) > 0
    b = int(np.argmax(snr[best[1], 1, :r.n_boxcars]))
    t_idx = int(n * 0.37) * L // n
    assert abs(int(idx[best[1], 1, b]) - t_idx) <= int(r.boxcar_length[b]), (idx[best[1], 1, b], t_idx)
    for j in range(len(dms)):
        r0 = res[j][0]
        assert sum(int(c) for c in r0.signal_count[:r0.n_boxcars]) == 0
    # the S/N peaks at d0
    peak = snr[:, 1, :].max(axis=1)
    assert int(np.argmax(peak)) == dms.index(d0)


@pytest.mark.parametrize("fmt", ["simple", "naocpsr_snap1"])
@pytest.mark.parametrize("name", ROW_CASES + ["long_n2_32768"])
def test_best_trial_outputs(ctx, name, fmt):
    """the best trial's h_series rows equal process_block's at that DM, d_spectrum of the last stream equals the
    spectrum of a sweep over [best DM] alone, and the call (which compares the re-run's header with its trial's) succeeds"""
    case = CASES[name]
    _, n, C_, _, _, dm = case
    L = n // 2 // C_
    cfg = _cfg(case, fmt)
    raw = _block(case, fmt, seed=42)
    pinned = _pinned(raw)
    dms = [0.0, 0.5 * dm, dm]
    streams = 2 if fmt == "naocpsr_snap1" else 1
    sentinel = np.float32(-12345.0)
    h_series = torch.full((streams, srtb_b200.MAX_BOXCARS, L), float(sentinel), dtype=torch.float32).pin_memory()
    res, _, best, h_series, d_spec = ctx.process_block_dm_sweep(cfg, pinned, raw.size, dms, outputs=True,
                                                                 h_series=h_series)
    torch.cuda.synchronize()
    assert best[0] == 2, "stream 0 carries the pulse at the case's DM"
    exact = _exact(case)
    for s in range(streams):
        cfg.dm = dms[best[s]]
        want = np.full((streams, srtb_b200.MAX_BOXCARS, L), sentinel, np.float32)
        block = ctx.process_block(cfg, pinned, raw.size, want, False)
        got = h_series[s].numpy()
        r = res[best[s]][s]
        if exact:
            assert _header_bytes(r) == _header_bytes(block[s])
            assert np.array_equal(got, want[s])
        else:
            positive = [b for b in range(r.n_boxcars) if r.signal_count[b] > 0]
            for b in range(srtb_b200.MAX_BOXCARS):
                if b in positive and block[s].signal_count[b] > 0:
                    m = int(r.series_length[b])
                    assert rel_l2(got[b, :m], want[s, b, :m]) < 2e-5
                elif b not in positive:
                    assert np.all(got[b] == sentinel)
        if s == streams - 1:
            ctx.process_block_dm_sweep(cfg, pinned, raw.size, [dms[best[s]]])
            alone = _from_device_ptr(ctx.sweep_spectrum_ptr(), C_ * L)
            mine = d_spec[s][:2 * C_ * L].cpu().numpy().view(np.complex64)
            assert np.array_equal(mine, alone)


def test_negative_block_leaves_series_untouched(ctx):
    """noise only: no trial is positive, and the pinned series buffer keeps its sentinel"""
    case = CASES["row16_4096"]
    _, n, C_, _, _, dm = case
    L = n // 2 // C_
    cfg = _cfg(case, snr=8.0)
    pinned = _pinned(_noise(n, 60))
    h_series = torch.full((1, srtb_b200.MAX_BOXCARS, L), 7.5, dtype=torch.float32).pin_memory()
    res, (snr, _), best, h_series, _ = ctx.process_block_dm_sweep(cfg, pinned, n, [0.0, 0.5 * dm, dm], outputs=True,
                                                                  h_series=h_series)
    for row in res:
        r = row[0]
        assert r.detect_enabled and sum(int(c) for c in r.signal_count[:r.n_boxcars]) == 0
    assert np.all(snr > 0) and np.all(snr < 8.0)
    assert torch.all(h_series == 7.5)
    assert best[0] == int(np.argmax(snr[:, 0, :].max(axis=1)))


def test_invalid_arguments(ctx):
    """each invalid argument returns E_INVALID and launches nothing"""
    case = CASES["row16_1024"]
    n = case[1]
    cfg = _cfg(case, "naocpsr_snap1")
    raw = _block(case, "naocpsr_snap1", seed=43)
    pinned = _pinned(raw)
    dms = (C.c_float * 2)(0.0, 1.0)
    res = (srtb_b200.DetectResult * 8)()
    spec = [torch.empty(n + 2 + 4, dtype=torch.float32, device="cuda") for _ in range(2)]
    lib, h = ctx.lib, ctx.h

    def outputs(d0, d1):
        o = srtb_b200.SweepOutputs()
        o.d_spectrum[0], o.d_spectrum[1] = d0, d1
        return o

    calls = [
        (cfg, pinned, dms, 2, res, None),
        (None, pinned, dms, 2, res, None),
        (cfg, None, dms, 2, res, None),
        (cfg, pinned, None, 2, res, None),
        (cfg, pinned, dms, 2, None, None),
        (cfg, pinned, dms, 0, res, None),
        (cfg, pinned, dms, 2, res, outputs(spec[0].data_ptr(), None)),
        (cfg, pinned, dms, 2, res, outputs(None, spec[1].data_ptr())),
        (cfg, pinned, dms, 2, res, outputs(spec[0].data_ptr() + 4, spec[1].data_ptr())),
        (cfg, pinned, dms, 2, res, outputs(spec[0].data_ptr(), spec[1].data_ptr() + 8)),
    ]
    for i, (c, bb, d, nd, r, o) in enumerate(calls):
        before = ctx.launch_count
        rc = lib.srtb_b200_process_block_dm_sweep_ex(h, C.byref(c) if c is not None else None,
                                                     srtb_b200._ptr(bb), raw.size, 0, d, nd, r,
                                                     C.byref(o) if o is not None else None)
        if i == 0:
            assert rc == 2
            continue
        assert rc == E_INVALID, (i, rc)
        assert ctx.launch_count == before, i
    assert lib.srtb_b200_process_block_dm_sweep_ex(None, C.byref(cfg), srtb_b200._ptr(pinned), raw.size, 0, dms, 2,
                                                   res, None) == E_INVALID


def test_executable_dm_list(tmp_path):
    """src/srtb_b200 with --dm_list over a file holding a pulse at d0 in stream 1: the S/N-versus-DM table of that
    stream peaks at d0, its .tim files name d0, and the best trial's spectrum is written"""
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    n, C_, f_low, bw, d0 = 1 << 22, 256, 1000.0, 64.0, 5.0
    raw = _snap1(_noise(n, 70), _with_pulse(n, 71, f_low, bw, d0))
    inp = tmp_path / "bb.bin"
    raw.tofile(inp)
    prefix = tmp_path / "cand_"
    cfg = tmp_path / "sweep.cfg"
    cfg.write_text(f"""# DM search
baseband_input_count = 2 ** 22
baseband_input_bits = -8
baseband_format_type = naocpsr_snap1
baseband_freq_low = {f_low}
baseband_bandwidth = {bw}
baseband_sample_rate = 2 * {bw} * 1e6
baseband_reserve_sample = 0
dm = 0
spectrum_channel_count = {C_}
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 8
signal_detect_max_boxcar_length = 256
input_file_path = {inp}
baseband_output_file_prefix = {prefix}
log_level = 3
""")
    # no core file if the executable aborts: a CUDA process's image is large
    r = subprocess.run([str(exe), "--config_file_name", str(cfg), "--dm_list", "0:10:2.5", "--ring_depth", "3"],
                       capture_output=True, text=True, timeout=300,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    assert "1 block(s) x 2 stream(s)" in r.stderr
    assert "5 trial DM(s)" in r.stderr and "ring_depth is ignored" in r.stderr, r.stderr[-3000:]
    csvs = sorted(tmp_path.glob("cand_*.1.dm_sweep.csv"))
    assert len(csvs) == 1, sorted(p.name for p in tmp_path.iterdir())
    assert not list(tmp_path.glob("cand_*.0.dm_sweep.csv"))  # stream 0 (noise) is negative
    lines = csvs[0].read_text().splitlines()
    assert lines[0] == "dm,detect_enabled,boxcar_length,series_length,signal_count,threshold,peak_snr,peak_index"
    rows = [ln.split(",") for ln in lines[1:]]
    n_boxcars = len({row[2] for row in rows})
    assert len(rows) == 5 * n_boxcars
    assert sorted({float(row[0]) for row in rows}) == [0.0, 2.5, 5.0, 7.5, 10.0]
    best = max(rows, key=lambda row: float(row[6]))
    assert float(best[0]) == d0
    stem = csvs[0].name.split(".")[0]
    tims = sorted(tmp_path.glob(f"{stem}.dm*.tim"))
    assert tims and all(p.name.startswith(f"{stem}.dm5.") for p in tims), [p.name for p in tims]
    npys = sorted(tmp_path.glob(f"{stem}.*.npy"))
    assert npys and np.load(npys[0]).shape == (C_, n // 2 // C_)
