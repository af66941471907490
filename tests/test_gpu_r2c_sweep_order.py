"""The config-#3 route that runs the R2C in two sweeps and leaves the spectrum in sweep order (2^25-point R2C, rows of
2^14: the raw 2^11-point column sweep, the paired 2^14-point row sweep with the split, and the whole-row waterfall kernel
reading its channels from that order), against float64 truth (DESIGN.md §4 parity policy)."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import srtb_b200  # noqa: E402
import detector_truth as dt  # noqa: E402
from test_gpu_parity import (REL_L2, _from_device_ptr, _host_floats, chain_truth_float64, make_block_config,  # noqa: E402
                             rel_l2, synth_baseband)

pytestmark = pytest.mark.gpu

N = 1 << 26          # samples per stream: M = 2^25 complex points = 2^11 rows of 2^14
C_ = 1 << 11
L = N // 2 // C_
P = C_
ZAP_MHZ = (1200.0, 1200.5)
F_LOW, BW, FS, DM = 1000.0, 500.0, 1e9, 562.05


def _block(seed):
    """two int8 streams in the naocpsr_snap1 layout (re0 im0 re1 im1 per point): the fused raw first sweep applies. No
    CW tone: SK would zap its channel, which the float64 chain below does not model"""
    s = [synth_baseband(N, seed=seed + i, tone=False, pulse=True) for i in range(2)]
    raw = np.empty(2 * N, np.int8)
    v = raw.reshape(-1, 2, 2)
    v[:, 0, :] = s[0].reshape(-1, 2)
    v[:, 1, :] = s[1].reshape(-1, 2)
    return raw, s


def _cfg(avg_thr, sk_thr=1.95, snr=50.0):
    return make_block_config(N, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, C_, DM, f_low=F_LOW, bw=BW, fs=FS, avg_thr=avg_thr,
                             sk_thr=sk_thr, snr=snr, maxbox=256, pairs=[ZAP_MHZ])


def _zap_bins():
    lo_hi = srtb_b200.rfi_range_to_bins(ZAP_MHZ[0], ZAP_MHZ[1], F_LOW, BW, N // 2)
    assert lo_hi is not None
    return [tuple(lo_hi)]


def _truth_detector(spec, cfg):
    reserved = srtb_b200.nsamps_reserved(N, C_, F_LOW, BW, FS, cfg.dm, True) // C_
    ts = dt.ts_count_for(L, reserved)
    A, zc = dt.column_power(spec, ts)
    return dt.truth_from_columns(A, C_, zc, cfg.signal_detect_signal_noise_threshold,
                                 cfg.signal_detect_channel_threshold, cfg.signal_detect_max_boxcar_length)


@pytest.fixture(scope="module")
def block():
    return _block(seed=2025)


def test_route_taken_and_spectrum_vs_float64(ctx, block):
    """both streams on two lanes: two R2C launches per stream instead of three sweeps and the column-0 fix-up, the
    dynamic spectrum within rel-L2 1e-5 and max-abs 1e-4 RMS of float64 (zap range included), the bins of the
    self-paired rows k1 = 0 and P/2 held to the same policy in the frequency domain, the detector within its bound"""
    raw, streams = block
    cfg = _cfg(avg_thr=1e9)
    pinned = torch.from_numpy(raw.view(np.uint8)).pin_memory()
    ctx.process_block(cfg, pinned, raw.size, None)   # tables and phase table built outside the counted call
    torch.cuda.synchronize()
    l0 = ctx.launch_count
    hs = np.full((2, srtb_b200.MAX_BOXCARS, L), np.nan, np.float32)
    res = ctx.process_block(cfg, pinned, raw.size, hs, copy_all=True)
    torch.cuda.synchronize()
    # per stream: raw 2^11-point column sweep, paired row sweep, one zap launch, whole-row kernel, two detector kernels
    # (the three-sweep plan launches three sweeps and the fix-up kernel: two more per stream)
    assert ctx.launch_count - l0 == 2 * 6
    zb = _zap_bins()
    for s in range(2):
        got = _from_device_ptr(ctx.block_spectrum_ptr(s), N // 2).reshape(C_, L)
        truth = chain_truth_float64(streams[s], cfg, zb)
        err = rel_l2(got, truth)
        rms = np.sqrt(np.mean(np.abs(truth) ** 2))
        print(f"stream {s}: rel-L2 vs float64 {err:.3e}, max-abs / RMS {np.abs(got - truth).max() / rms:.3e}")
        assert err < REL_L2
        assert np.abs(got - truth).max() < 1e-4 * rms
        # frequency domain: bins k = k1 + P k2 of the self-paired rows (and a generic pair) of the row sweep
        G = np.fft.fft(got.astype(np.complex128), axis=1).reshape(-1)
        T = np.fft.fft(truth, axis=1).reshape(-1)
        for k1 in (0, P // 2, 1, P - 1, 777):
            idx = k1 + P * np.arange(N // 2 // P)
            e = np.linalg.norm(G[idx] - T[idx]) / np.linalg.norm(T[idx])
            assert e < REL_L2, (s, k1, e)
        lo, hi = zb[0]
        assert np.abs(G[lo:hi + 1]).max() < 1e-4 * np.sqrt(np.mean(np.abs(T) ** 2))
        t = _truth_detector(got, cfg)
        rows = list(range(t.n_boxcars)) if t.detect_enabled else [0]
        dt.compare(res[s], hs[s], t, rows=rows)


def test_s1_mean_through_zap_decisions(ctx, block):
    """the row sweep's mean of |X|^2 decides the s1 zap (above 1.5 x mean): every bin the GPU zapped or kept against
    the float64 decision lies within 2e-6 of the float64 threshold, so the mean agrees to about 1e-6"""
    raw, streams = block
    cfg = _cfg(avg_thr=1.5)
    ctx.process_block(cfg, torch.from_numpy(raw.view(np.uint8)).pin_memory(), raw.size, None)
    torch.cuda.synchronize()
    for s in range(2):
        got = _from_device_ptr(ctx.block_spectrum_ptr(s), N // 2).reshape(C_, L)
        Y = np.fft.fft(got.astype(np.complex128), axis=1).reshape(-1)
        X = np.fft.rfft(streams[s].astype(np.float64))[:N // 2]
        pw = np.abs(X) ** 2
        thr = np.float64(np.float32(1.5)) * pw.mean()
        coef = np.float64(srtb_b200.norm_coefficient(N // 2, C_))
        zapped = np.abs(Y) < 0.5 * coef * L * np.abs(X)   # kept bins come back with |Y| = coef L |X|
        lo, hi = _zap_bins()[0]
        expect = pw > thr
        expect[lo:hi + 1] = True
        differ = np.nonzero(zapped != expect)[0]
        print(f"stream {s}: {expect.mean():.3f} of bins zapped, {differ.size} decisions differ from float64")
        assert np.all(np.abs(pw[differ] / thr - 1) < 2e-6), (s, differ[:10], pw[differ[:10]] / thr)


def _digest(ctx, res, streams=2):
    h = hashlib.sha256()
    for s in range(streams):
        h.update(_from_device_ptr(ctx.block_spectrum_ptr(s), N // 2).tobytes())
        h.update(repr((int(res[s].zero_count), [int(c) for c in res[s].signal_count[:res[s].n_boxcars]])).encode())
    return h.hexdigest()


def test_one_lane_equals_two_lanes(ctx, block, tmp_path):
    """SRTB_B200_LANES=1 (both streams on one CUDA stream, one scratch, one ticket) in a child process gives the same
    spectra and headers, bit for bit, as two lanes"""
    raw, _ = block
    cfg = _cfg(avg_thr=1.5, sk_thr=1.05, snr=8.0)
    res = ctx.process_block(cfg, torch.from_numpy(raw.view(np.uint8)).pin_memory(), raw.size, None)
    torch.cuda.synchronize()
    mine = _digest(ctx, res)
    path = tmp_path / "raw.npy"
    np.save(path, raw)
    code = ("import os, sys, numpy as np, torch; import srtb_b200;"
            "from test_gpu_r2c_sweep_order import _cfg, _digest;"
            "raw = np.load(%r); ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream);"
            "cfg = _cfg(avg_thr=1.5, sk_thr=1.05, snr=8.0);"
            "r = ctx.process_block(cfg, torch.from_numpy(raw.view(np.uint8)).pin_memory(), raw.size, None);"
            "torch.cuda.synchronize(); print('DIGEST', _digest(ctx, r))") % str(path)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900,
                         env={**os.environ, "SRTB_B200_LANES": "1", "PYTHONPATH": os.pathsep.join(sys.path)})
    assert out.returncode == 0, out.stderr[-2000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("DIGEST")][-1]
    assert line.split()[1] == mine


def test_ring_with_caller_buffers_equals_process_block(ctx, block):
    """the ring with caller-owned spectrum and series buffers leaves what process_block leaves, on this route"""
    raw, _ = block
    cfg = _cfg(avg_thr=1.5, sk_thr=1.05, snr=8.0)
    b = torch.from_numpy(raw.view(np.uint8)).pin_memory()
    hs = np.zeros((2, srtb_b200.MAX_BOXCARS, L), np.float32)
    expect = ctx.process_block(cfg, b, raw.size, hs, copy_all=True)
    torch.cuda.synchronize()
    espec = [_from_device_ptr(ctx.block_spectrum_ptr(s), N // 2) for s in range(2)]
    specs = [torch.empty(N + 2, dtype=torch.float32, device="cuda") for _ in range(2)]
    ser = torch.zeros(2 * srtb_b200.MAX_BOXCARS * L, dtype=torch.float32).pin_memory()
    t = ctx.submit_block_ex(cfg, b, raw.size, False, specs, ser)
    res, series_ptr, spec_ptrs = ctx.collect_block_ex(t)
    assert [int(p) for p in spec_ptrs] == [s.data_ptr() for s in specs]
    got_series = _host_floats(series_ptr, 2 * srtb_b200.MAX_BOXCARS * L).reshape(2, -1, L)
    for s in range(2):
        assert np.array_equal(_from_device_ptr(spec_ptrs[s], N // 2), espec[s]), f"stream {s}: spectrum differs"
        assert list(res[s].signal_count[:res[s].n_boxcars]) == list(expect[s].signal_count[:expect[s].n_boxcars])
        for k in range(res[s].n_boxcars):
            if res[s].signal_count[k] > 0:
                ln = int(res[s].series_length[k])
                assert np.array_equal(got_series[s, k, :ln], hs[s, k, :ln])
