"""The single-pulse detector on the GPU against its float64 truth (detector_truth.py) on every path that feeds it.

Per-pipe signal_detect and signal_detect_v1 run at the scan, chunk and boxcar edges of test_detector_truth's geometries.
The block path runs each producer of the partial column sums, at a DM and with reserve_sample so that the detector
trims ts_count below L, with an SK-zapped channel: the truth there is computed from the dynamic spectrum the same call
left on the device, so a dropped column, a wrongly trimmed cell or a zapped row that is still summed fails.

Every header field is checked: the exact ones for equality, variance and threshold within their bound, signal counts
within [#(S > thr + m), #(S >= thr - m)]. Host series buffers are filled with NaN first: rows with a positive count
must hold the device series, every other row must stay NaN.

Every case runs under torch.profiler; the last test checks that each case launched the kernel that feeds its detector,
plus colsum_final_scan_kernel and detect_boxcar_kernel.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import detector_truth as dt  # noqa: E402
import srtb_b200  # noqa: E402
from test_detector_truth import CHAN_THR, PIPE_CASES, SNR, V1_CASES, pipe_spectrum, v1_spectrum  # noqa: E402
from test_fft_kernel_coverage import normalise  # noqa: E402
from test_gpu_parity import make_block_config  # noqa: E402

MAXB = srtb_b200.MAX_BOXCARS
LAUNCHED = {}        # case id -> base names of the library kernels it launched
PROFILER_SEES_KERNELS = []
WORST = {}           # route -> largest error / bound seen, per output
TAIL = {"colsum_final_scan_kernel", "detect_boxcar_kernel"}


@pytest.fixture(scope="module")
def dctx():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    torch.cuda.set_device(0)
    c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _record_kernels(request):
    """runs the case under torch.profiler (CUDA activities) and records the kernels it launched; one torch kernel is
    launched in the window so that a profiler that records nothing can be told from a route that launched nothing"""
    from torch.profiler import ProfilerActivity, profile
    if request.node.name == "test_every_case_launched_its_detector_feeder":
        yield
        return
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            yield
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        PROFILER_SEES_KERNELS.append(bool(names))
        LAUNCHED[request.node.name] = {normalise(n).split("<")[0] for n in names if "srtb_b200" in n}
    finally:
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------- helpers
def _device_copy(ptr, n_complex):
    """a torch copy of n complex64 at a raw device pointer"""
    cudart = C.CDLL("libcudart.so")
    cudart.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    out = torch.empty(n_complex, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    assert cudart.cudaMemcpy(out.data_ptr(), ptr, out.numel() * 8, 3) == 0   # device to device
    return out


def _truth(y, ts_count, snr=SNR, chan_thr=CHAN_THR, max_boxcar=1 << 30):
    """float64 truth of the detector on y: [rows][cols] complex64 on the device whose first ts_count columns are summed
    over rows (the per-pipe / block layout [C][L]; the v1 layout passes the transposed view). The column sums are
    formed on the device in float64, rows in chunks."""
    A = torch.zeros(ts_count, dtype=torch.float64, device="cuda")
    step = max(1, (1 << 24) // y.shape[1])
    for r in range(0, y.shape[0], step):
        A += torch.view_as_real(y[r:r + step, :ts_count]).double().pow(2).sum(dim=(0, 2))
    first = y[:, 0]
    zc = int(((first.real * first.real + first.imag * first.imag) == 0).sum())   # fp32, as the reference
    return dt.truth_from_columns(A.cpu().numpy(), y.shape[0], zc, snr, chan_thr, max_boxcar)


def _nan_series(rows, L, pinned=False):
    if pinned:
        return torch.full((rows, L), float("nan"), dtype=torch.float32).pin_memory()
    return np.full((rows, L), np.nan, np.float32)


def _record(route, worst):
    w = WORST.setdefault(route, {k: 0.0 for k in worst})
    for k, v in worst.items():
        w[k] = max(w[k], v)


def _check_full(route, res, h, t):
    """a result fetched with copy_all: header against the truth, every copied row within its bound, the rest NaN"""
    rows = list(range(t.n_boxcars)) if t.detect_enabled else [0]
    _record(route, dt.compare(res, h, t, rows=rows))
    for b in range(h.shape[0]):
        n = (t.series_length[b] if t.detect_enabled else t.time_series_count) if b in rows else 0
        assert np.isnan(h[b, n:]).all(), f"row {b}: written past its series ({n} values)"


def _check_positive_rows(route, res, h, t, h_all=None):
    """a result fetched without copy_all (or written by the ring): header against the truth, every row with a positive
    count within its bound (and bit-equal to h_all, the same call with copy_all, when given), every other row NaN"""
    _record(route, dt.compare(res, None, t))
    for b in range(h.shape[0]):
        if b < t.n_boxcars and res.signal_count[b] > 0:
            n = t.series_length[b]
            _record(route, dt.compare(res, h, t, rows=[b]))
            if h_all is not None:
                assert np.array_equal(h[b, :n].view(np.uint32), h_all[b, :n].view(np.uint32)), f"row {b} differs"
            assert np.isnan(h[b, n:]).all(), f"row {b}: written past its series"
        else:
            assert np.isnan(h[b]).all(), f"row {b} (count 0 or no boxcar) was written"


# ----------------------------------------------------------------------------- per-pipe signal_detect
@pytest.mark.parametrize("C_,L,reserved,maxbox", PIPE_CASES)
def test_signal_detect_edges(dctx, C_, L, reserved, maxbox):
    x = pipe_spectrum(C_, L, seed=C_ * 7919 + L)
    d = torch.from_numpy(x.reshape(-1)).cuda()
    t = _truth(d.view(C_, L), dt.ts_count_for(L, reserved), max_boxcar=maxbox)
    h1 = _nan_series(MAXB, L)
    r1 = dctx.signal_detect(d, L, C_, reserved, SNR, CHAN_THR, maxbox, h1, copy_all=True)
    _check_full("signal_detect", r1, h1, t)
    h2 = _nan_series(MAXB, L)
    r2 = dctx.signal_detect(d, L, C_, reserved, SNR, CHAN_THR, maxbox, h2, copy_all=False)
    assert bytes(r1) == bytes(r2), "the same input gave another header"
    _check_positive_rows("signal_detect", r2, h2, t, h_all=h1)


@pytest.mark.parametrize("zero_rows", [8, 9])
def test_channel_threshold_boundary(dctx, zero_rows):
    """float(0.9) * float(10) is 9 in fp32: 8 zeroed channels of 10 leave detection on, 9 switch it off"""
    C_, L = 10, 256
    x = pipe_spectrum(C_, L, seed=zero_rows)
    x[:zero_rows] = 0
    d = torch.from_numpy(x.reshape(-1)).cuda()
    t = _truth(d.view(C_, L), L, max_boxcar=64)
    h = _nan_series(MAXB, L)
    res = dctx.signal_detect(d, L, C_, 0, SNR, CHAN_THR, 64, h, copy_all=True)
    assert res.zero_count == zero_rows and bool(res.detect_enabled) == (zero_rows == 8)
    _check_full("signal_detect", res, h, t)


def test_constant_rows_zero_variance(dctx):
    """rows constant in time with powers 1, 4, 9: column sums, mean and d = 0 are exact, so var = thr = 0 and no sample
    may count (S > 0 is false everywhere; S >= 0 would count all of them)"""
    C_, L = 10, 5000
    x = np.repeat((np.arange(C_) % 3 + 1).astype(np.complex64)[:, None], L, axis=1)
    h = _nan_series(MAXB, L)
    res = dctx.signal_detect(torch.from_numpy(x.reshape(-1)).cuda(), L, C_, 0, SNR, CHAN_THR, 64, h, copy_all=True)
    assert res.detect_enabled == 1 and res.n_boxcars == 7
    for b in range(res.n_boxcars):
        n = int(res.series_length[b])
        assert res.variance[b] == 0 and res.threshold[b] == 0 and res.signal_count[b] == 0
        assert not h[b, :n].any() and not np.isnan(h[b, :n]).any()
        assert np.isnan(h[b, n:]).all()
    assert np.isnan(h[res.n_boxcars:]).all()


def test_all_zero_spectrum_is_disabled_and_copy_all_returns_row_0(dctx):
    C_, L = 64, 1000
    d = torch.zeros(C_ * L, dtype=torch.complex64, device="cuda")
    h = _nan_series(MAXB, L)
    res = dctx.signal_detect(d, L, C_, 3, SNR, CHAN_THR, 64, h, copy_all=True)
    assert res.zero_count == C_ and res.detect_enabled == 0 and res.n_boxcars == 0
    assert res.time_series_count == L - 3
    assert not h[0, :L - 3].any() and np.isnan(h[0, L - 3:]).all() and np.isnan(h[1:]).all()
    h2 = _nan_series(MAXB, L)
    dctx.signal_detect(d, L, C_, 3, SNR, CHAN_THR, 64, h2, copy_all=False)
    assert np.isnan(h2).all()


def test_large_grid_after_a_one_cta_call_equals_a_fresh_context(dctx):
    """the last-CTA ticket and the zero count are reset by the call that used them: a call on 132 CTAs after one on a
    single CTA gives the bits a fresh context gives"""
    small = torch.from_numpy(pipe_spectrum(3000, 32, seed=1).reshape(-1)).cuda()
    big = torch.from_numpy(pipe_spectrum(33, 20000, seed=2).reshape(-1)).cuda()
    dctx.signal_detect(small, 32, 3000, 0, SNR, CHAN_THR, 8)
    h_a = _nan_series(MAXB, 20000)
    r_a = dctx.signal_detect(big, 20000, 33, 0, SNR, CHAN_THR, 1024, h_a, copy_all=True)
    fresh = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        h_b = _nan_series(MAXB, 20000)
        r_b = fresh.signal_detect(big, 20000, 33, 0, SNR, CHAN_THR, 1024, h_b, copy_all=True)
    finally:
        fresh.close()
    assert bytes(r_a) == bytes(r_b)
    assert np.array_equal(h_a.view(np.uint32), h_b.view(np.uint32))


# ----------------------------------------------------------------------------- v1 ([time][frequency])
@pytest.mark.parametrize("nt,nf,maxbox", V1_CASES)
def test_signal_detect_v1_edges(dctx, nt, nf, maxbox):
    """truth from the spectrum the call's SK v1 left behind; the zero count runs over the first spectrum (more than
    1024 channels with batch_size <= 32: its grid-stride loop)"""
    x = v1_spectrum(nt, nf, seed=nt * 31 + nf)
    d = torch.from_numpy(x.reshape(-1)).cuda()
    h = _nan_series(MAXB, nt)
    res = dctx.signal_detect_v1(d, nf, nt, 1.4, SNR, CHAN_THR, maxbox, h, copy_all=True)
    y = d.view(nt, nf)
    assert not y[:, 5].any() and res.zero_count >= 2 + (nf > 1024)
    _check_full("signal_detect_v1", res, h, _truth(y.t(), nt, max_boxcar=maxbox))


# ----------------------------------------------------------------------------- block path
D = 4.148808e3


def _block(L, C_, seed, maxbox=1 << 20, fmt=srtb_b200.FORMAT_SIMPLE, streams=1):
    """config and 8-bit baseband of a block with rows of L: noise, a strong steady tone (SK zaps its channel; the s1
    threshold is out of the way), a weak broadband burst (+30% over L/4 time bins: the chirp of the block's DM smears
    it over L/8 bins, and the wide boxcars still find it), and a DM with reserve_sample that reserves about a quarter
    of every row"""
    n = 2 * C_ * L
    f_lo, bw, fs = 1000.0, 500.0, 1e9
    dm = n / (16 * fs * D * (1 / f_lo ** 2 - 1 / (f_lo + bw) ** 2))
    cfg = make_block_config(n, -8, fmt, C_, dm, f_low=f_lo, bw=bw, fs=fs, avg_thr=1e9, sk_thr=1.5, snr=SNR,
                            chan_thr=CHAN_THR, maxbox=maxbox)
    cfg.baseband_reserve_sample = 1
    reserved = srtb_b200.nsamps_reserved(n, C_, f_lo, bw, fs, cfg.dm, True) // C_
    assert 0 < reserved < L
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    out = []
    for s in range(streams):
        v = rng.standard_normal(n) * 20 + 50 * np.cos(2 * np.pi * (0.1185 + 0.01 * s) * t)
        v[n // 4:n // 4 + n // 8] *= 1.3
        out.append(np.clip(np.round(v), -127, 127).astype(np.int8))
    if streams == 1:
        raw = out[0]
    else:   # naocpsr_snap1: two samples of stream 0, then two of stream 1
        raw = np.empty(2 * n, np.int8)
        raw.reshape(-1, 4)[:, 0:2] = out[0].reshape(-1, 2)
        raw.reshape(-1, 4)[:, 2:4] = out[1].reshape(-1, 2)
    return cfg, torch.from_numpy(raw.view(np.uint8).copy()).cuda(), L - reserved


def _block_truth(ptr, C_, L, ts_count, maxbox):
    y = _device_copy(ptr, C_ * L).view(C_, L)
    zapped = int((y.abs().amax(dim=1) == 0).sum())
    assert zapped >= 1, "no channel was zapped: the tone did not reach SK"
    return _truth(y, ts_count, max_boxcar=maxbox)


# case id, L, C, kernels that feed the detector on that route
BLOCK_CASES = [
    ("L256", 256, 64, {"colsum_partial_kernel", "sk_kernel"}),          # unfused: SK, then detect_enqueue
    ("L512", 512, 64, {"fft_row_tma_kernel"}),                           # eight-point SK row kernel
    ("L1024", 1024, 64, {"fft_row16_tma_kernel"}),
    ("L4096", 4096, 64, {"fft_row16_tma_kernel"}),
    ("L8192", 8192, 64, {"fft_bigrow_kernel"}),
    ("L16384_C16", 16384, 16, {"fft_bigrow_kernel"}),
    ("L32768", 1 << 15, 32, {"sk_decide_kernel", "colsum_partial_kernel"}),
    ("L262144", 1 << 18, 8, {"sk_decide_kernel", "colsum_partial_kernel"}),
    ("L524288", 1 << 19, 4, {"colsum_partial_kernel", "sk_kernel"}),   # unfused again above 2^18
]
FEEDERS = {}         # test node name -> kernels it must have launched


@pytest.mark.parametrize("case", BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_block_path_feeders(request, dctx, case):
    name, L, C_, feeders = case
    FEEDERS[request.node.name] = feeders
    maxbox = 100 if L == 4096 else 1 << 20
    cfg, d, ts = _block(L, C_, seed=L + C_, maxbox=maxbox)
    n = cfg.baseband_input_count
    h1 = _nan_series(MAXB, L)
    r1 = dctx.process_block(cfg, d, n, h1, copy_all=True, on_device=True)[0]
    t = _block_truth(dctx.block_spectrum_ptr(0), C_, L, ts, maxbox)
    assert t.detect_enabled and r1.time_series_count == ts
    _check_full(f"block {name}", r1, h1, t)
    h2 = _nan_series(MAXB, L)
    r2 = dctx.process_block(cfg, d, n, h2, copy_all=False, on_device=True)[0]
    assert bytes(r1) == bytes(r2), "the same block gave another header"
    _check_positive_rows(f"block {name}", r2, h2, t, h_all=h1)


def test_block_two_streams(request, dctx):
    """the second stream runs on the context's second lane, with that lane's partial, scan and ticket buffers"""
    FEEDERS[request.node.name] = {"fft_row16_tma_kernel"}
    L, C_ = 4096, 64
    cfg, d, ts = _block(L, C_, seed=11, fmt=srtb_b200.FORMAT_NAOCPSR_SNAP1, streams=2)
    h = _nan_series(2 * MAXB, L)
    res = dctx.process_block(cfg, d, 4 * C_ * L, h, copy_all=True, on_device=True)
    assert len(res) == 2
    for s in range(2):
        t = _block_truth(dctx.block_spectrum_ptr(s), C_, L, ts, 1 << 20)
        _check_full("block two streams", res[s], h[s * MAXB:(s + 1) * MAXB], t)


def test_dm_sweep_last_trial(request, dctx):
    FEEDERS[request.node.name] = {"fft_bigrow_kernel"}
    L, C_ = 8192, 64
    cfg, d, _ = _block(L, C_, seed=12)
    n = cfg.baseband_input_count
    dms = [cfg.dm, cfg.dm / 3]
    sweep = dctx.process_block_dm_sweep(cfg, d, n, dms, on_device=True)
    ts = L - srtb_b200.nsamps_reserved(n, C_, 1000.0, 500.0, 1e9, dms[-1], True) // C_
    t = _block_truth(dctx.sweep_spectrum_ptr(), C_, L, ts, 1 << 20)
    _record("dm sweep", dt.compare(sweep[-1][0], None, t))


def test_ring_with_caller_series_and_changing_rows(request, dctx):
    """three blocks in flight through the ring, rows of 2^14 -> 2^12 -> 2^14, each with its own device spectrum and
    pinned series buffer: the detector kernel writes the positive series straight into it and nothing else"""
    FEEDERS[request.node.name] = {"fft_bigrow_kernel", "fft_row16_tma_kernel"}
    blocks = []
    for i, (L, C_) in enumerate([(1 << 14, 32), (1 << 12, 128), (1 << 14, 32)]):
        cfg, d, ts = _block(L, C_, seed=20 + i)
        spec = torch.empty(cfg.baseband_input_count + 2, dtype=torch.float32, device="cuda")
        hs = _nan_series(MAXB, L, pinned=True)
        blocks.append((cfg, d, ts, L, C_, spec, hs))
    tickets = [dctx.submit_block_ex(cfg, d, cfg.baseband_input_count, True, [spec], hs)
               for cfg, d, _, _, _, spec, hs in blocks]
    positive = zero = 0
    for tk, (cfg, _, ts, L, C_, spec, hs) in zip(tickets, blocks):
        res, series_ptr, spec_ptrs = dctx.collect_block_ex(tk)
        assert series_ptr == hs.data_ptr() and spec_ptrs[0] == spec.data_ptr()
        t = _block_truth(spec_ptrs[0], C_, L, ts, 1 << 20)
        _check_positive_rows("ring", res[0], hs.numpy(), t)
        counts = [int(res[0].signal_count[b]) for b in range(res[0].n_boxcars)]
        positive += sum(c > 0 for c in counts)
        zero += sum(c == 0 for c in counts)
    assert positive > 0 and zero > 0, "the ring run should have rows of both kinds"


# ----------------------------------------------------------------------------- routes and report
def test_every_case_launched_its_detector_feeder(request):
    if not LAUNCHED:
        pytest.skip("no case of this module ran")
    if not any(PROFILER_SEES_KERNELS):
        pytest.skip("torch.profiler recorded no CUDA kernel at all, not even torch's own")
    missing = []
    for case, kernels in LAUNCHED.items():
        need = set(TAIL)
        if case.startswith("test_signal_detect_edges") or case.startswith("test_channel_threshold"):
            need.add("colsum_partial_kernel")
        if case.startswith("test_signal_detect_v1_edges"):
            need.add("rowsum_norm_kernel")
        need |= FEEDERS.get(case, set())
        if not need <= kernels:
            missing.append(f"{case}: {sorted(need - kernels)} not launched")
    assert not missing, "\n".join(missing)
    print("\nlargest error / bound per route:")
    for route, w in sorted(WORST.items()):
        print(f"  {route:28s} " + "  ".join(f"{k} {v:.3g}" for k, v in w.items()))
