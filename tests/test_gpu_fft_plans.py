"""Every FFT plan, aligned and at +8 bytes, against float64; the element-wise stages and the block path on pointers
that are only 8-byte (complex64) or 1-byte (baseband) aligned.

A complex64 view that starts at an odd element (x[1:]) is 8-byte aligned: the FFT then leaves the TMA-fed passes for
the plain-load row, column and transposing passes, lengths 2^13 / 2^14 leave the whole-row kernel for the two-sweep
plan, and 2^27 .. 2^30 take three sweeps instead of four. The element-wise stages take their 8-byte loops.

Every case runs under torch.profiler; test_fft_kernel_coverage.KERNEL_CASES names, for every FFT-engine kernel of the
library, the case below that must launch it, and the last test checks that it did (a +8 case that silently took a
TMA route fails there).

Tolerances are those of test_gpu_parity.py: rel-L2 <= 1e-5 against float64, and the per-element bound
clamp(eps * n / 2, 1e-5, 0.05) of max |error| over max |truth| (the reference's FFT test). Above 2^27 points the
truth is a sum of 64 complex tones at random integer bins, whose spectrum is known exactly.
"""

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import srtb_b200  # noqa: E402
from test_chirp_newton import GPU_CASES  # noqa: E402
from test_fft_kernel_coverage import KERNEL_CASES, normalise  # noqa: E402
from test_gpu_parity import (BORDER, _compare_detect, _from_device_ptr, _refft_layout_block, _spectrum,  # noqa: E402
                             chain_truth_float64, make_block_config, rel_l2, synth_baseband)

REL_L2 = 1e-5
E_INVALID, E_SIZE = -1, -2
LAUNCHED = {}        # case id -> normalised names of the kernels it launched
PROFILER_SEES_KERNELS = []


@pytest.fixture(scope="module")
def fctx():
    """a context of this module's own: the 8 GiB of FFT scratch at 2^30 goes with it at module end"""
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
    if request.node.name == "test_every_listed_kernel_was_launched":
        yield
        return
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            yield
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        ours = {normalise(n) for n in names if "srtb_b200" in n or "tiny_fft_kernel" in n}
        PROFILER_SEES_KERNELS.append(bool(names))
        LAUNCHED[request.node.name] = ours
        print(f"\n  launched by {request.node.name}: {' '.join(sorted(ours))}")
    finally:
        torch.cuda.empty_cache()   # gigabytes of cached test buffers would starve the library's own cudaMalloc


# ----------------------------------------------------------------------------- helpers
def _view(n_complex, off_bytes, dtype=torch.complex64):
    """a device view of n_complex elements whose address is off_bytes past a 256-byte aligned allocation"""
    esz = torch.empty(0, dtype=dtype).element_size()
    assert off_bytes % esz == 0
    base = torch.zeros(n_complex + off_bytes // esz + 1, dtype=dtype, device="cuda")
    v = base[off_bytes // esz:off_bytes // esz + n_complex]
    assert v.data_ptr() % 16 == off_bytes % 16
    return v


def _dev_rel_l2(got, truth):
    got = got.to(torch.complex128)
    return float(((got - truth).abs().pow(2).sum() / truth.abs().pow(2).sum()).sqrt())


def _elem_bound(n):
    return float(np.clip(np.finfo(np.float32).eps * n / 2, 1e-5, 0.05))


def _uniform(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.view_as_complex(torch.rand(*shape, 2, device="cuda", generator=g) * 2 - 1)


def _tones(n, bins, amps, out, real=False):
    """out[t] = sum_j amps[j] exp(2 pi i bins[j] t / n) (or its real part), evaluated in float64 as the product of a
    [n/w][64] and a [64][w] matrix (t = t_hi w + t_lo) with exact integer phases, rows in chunks"""
    w = 1 << ((n.bit_length() - 1 + 1) // 2)
    h = n // w
    b = torch.tensor(bins, dtype=torch.int64, device="cuda")
    a = torch.tensor(amps, dtype=torch.complex128, device="cuda")
    tl = torch.arange(w, dtype=torch.int64, device="cuda")
    th = torch.arange(h, dtype=torch.int64, device="cuda")
    def cis(m):  # exp(2 pi i m / n) for integer m in [0, n)
        ang = m.to(torch.float64) * (2 * np.pi / n)
        return torch.complex(torch.cos(ang), torch.sin(ang))
    B = cis((b[:, None] * tl[None, :]) % n)
    A = a[None, :] * cis((((b * w) % n)[None, :] * th[:, None]) % n)
    o = out.view(h, w)
    rows = max(1, (1 << 27) // w)
    for r in range(0, h, rows):
        blk = A[r:r + rows] @ B
        o[r:r + rows] = blk.real.to(torch.float32) if real else blk.to(torch.complex64)
        del blk


def _tone_errors(y, tone_bins, tone_vals):
    """rel-L2 and max-error ratio of a spectrum y (complex64 on the device) whose truth is tone_vals at tone_bins and
    zero elsewhere; the off-tone energy is summed with the tone bins zeroed (no cancellation)"""
    idx = torch.tensor(tone_bins, dtype=torch.int64, device="cuda")
    t = torch.tensor(tone_vals, dtype=torch.complex128, device="cuda")
    at = y[idx].to(torch.complex128)
    y[idx] = 0
    off2, offmax = 0.0, 0.0
    chunk = 1 << 26
    for s in range(0, y.numel(), chunk):
        m = y[s:s + chunk].abs().double()
        off2 += float(m.pow(2).sum())
        offmax = max(offmax, float(m.max()))
    err2 = off2 + float((at - t).abs().pow(2).sum())
    rel = np.sqrt(err2 / float(t.abs().pow(2).sum()))
    emax = max(offmax, float((at - t).abs().max())) / float(t.abs().max())
    return rel, emax


def _tone_plan(n, seed, count=64, lo=0, hi=None):
    rng = np.random.default_rng(seed)
    bins = rng.choice(np.arange(lo, hi if hi is not None else n), count, replace=False).astype(np.int64)
    amps = rng.uniform(0.5, 2.0, count) * np.exp(2j * np.pi * rng.uniform(0, 1, count))
    return bins, amps


def _device_spectrum(ptr, n_complex):
    """device copy of n_complex complex64 at a device pointer the library returned"""
    import ctypes as CT
    out = torch.empty(n_complex, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    cudart = CT.CDLL("libcudart.so")
    cudart.cudaMemcpy.argtypes = [CT.c_void_p, CT.c_void_p, CT.c_size_t, CT.c_int]
    assert cudart.cudaMemcpy(out.data_ptr(), ptr, out.numel() * 8, 3) == 0
    return out


def _chain_truth_dev(samples, cfg, dm):
    """test_gpu_parity.chain_truth_float64 on the device (float64 torch), for blocks too long for numpy:
    R2C -> s1 -> chirp at `dm` -> waterfall, with the reference's float32 parameter roundings"""
    n = cfg.baseband_input_count
    nc = n // 2
    C_ = min(cfg.spectrum_channel_count, nc)
    X = torch.fft.rfft(samples.to(torch.float64))[:nc]
    pw = X.abs() ** 2
    coef = float(srtb_b200.norm_coefficient(nc, cfg.spectrum_channel_count))
    X = torch.where(pw > float(np.float32(cfg.mitigate_rfi_average_method_threshold)) * pw.mean(), 0, X * coef)
    del pw
    f_min, bw = np.float32(cfg.baseband_freq_low), np.float32(cfg.baseband_bandwidth)
    f_c = float(np.float32(f_min + bw))
    df = float(np.float32(bw / np.float32(nc)))
    f = float(f_min) + df * torch.arange(nc, dtype=torch.float64, device="cuda")
    k = (4.148808e3 * 1e6) * float(np.float32(dm)) / f * ((f - f_c) / f_c) ** 2
    ang = -2 * np.pi * (k - torch.trunc(k))
    del f, k
    X = X * torch.complex(torch.cos(ang), torch.sin(ang))
    return torch.fft.ifft(X.view(C_, nc // C_), dim=1, norm="forward")


def _spectrum_vs_truth(label, ptr, truth):
    """rel-L2 of a block's dynamic spectrum against float64 over the channels the block kept (SK may zap the channel
    that holds the DC level of unsigned samples)"""
    C_, L = truth.shape
    got = _device_spectrum(ptr, C_ * L).view(C_, L)
    keep = (got != 0).any(dim=1)
    assert int(keep.sum()) >= C_ - 1, f"{label}: {C_ - int(keep.sum())} channels zapped"
    err = _dev_rel_l2(got[keep], truth[keep])
    print(f"{label}: rel-L2 {err:.3e} over {int(keep.sum())} of {C_} channels")
    assert err < REL_L2, f"{label}: rel-L2 {err:.3e}"


def _err_code(fn):
    with pytest.raises(srtb_b200.SrtbError) as e:
        fn()
    return e.value.code


# ----------------------------------------------------------------------------- C2C
def _c2c_cases():
    out = []
    for k in range(1, 28):
        batch = (5 if k % 2 else 3) if k <= 20 else 1
        for off in (0, 8):
            out.append(pytest.param(k, batch, off, id=f"k{k}-b{batch}-off{off}"))
    for k in (21, 27):
        for off in (0, 8):
            out.append(pytest.param(k, 3, off, id=f"k{k}-b3-off{off}"))
    return out


@pytest.mark.parametrize("direction", [1, -1], ids=["fwd", "bwd"])
@pytest.mark.parametrize("k,batch,off", _c2c_cases())
def test_c2c_vs_float64(fctx, k, batch, off, direction):
    n = 1 << k
    x = _uniform((batch, n), seed=k * 131 + batch * 7 + off)
    v = _view(batch * n, off)
    v.copy_(x.reshape(-1))
    fctx.fft_c2c(v, n, batch, direction)
    x128 = x.to(torch.complex128)
    truth = torch.fft.fft(x128, dim=-1) if direction == 1 else torch.fft.ifft(x128, dim=-1, norm="forward")
    del x128
    got = v.view(batch, n)
    err = _dev_rel_l2(got, truth)
    emax = float((got.to(torch.complex128) - truth).abs().max() / truth.abs().max())
    print(f"c2c n=2^{k} batch={batch} +{off} dir={direction}: rel-L2 {err:.3e}, max {emax:.3e}")
    assert err < REL_L2
    assert emax < _elem_bound(n)


@pytest.mark.parametrize("direction", [1, -1], ids=["fwd", "bwd"])
@pytest.mark.parametrize("off", [0, 8], ids=["off0", "off8"])
@pytest.mark.parametrize("k", [28, 29, 30])
def test_c2c_tones_full_length(fctx, k, off, direction):
    n = 1 << k
    bins, amps = _tone_plan(n, seed=k * 10 + off)
    v = _view(n, off)
    _tones(n, bins, amps, v)
    fctx.fft_c2c(v, n, 1, direction)
    torch.cuda.synchronize()
    out_bins = bins if direction == 1 else (-bins) % n
    err, emax = _tone_errors(v, out_bins, amps * n)
    print(f"c2c tones n=2^{k} +{off} dir={direction}: rel-L2 {err:.3e}, max {emax:.3e}")
    assert err < REL_L2
    assert emax < _elem_bound(n)


@pytest.mark.parametrize("off", [0, 8], ids=["off0", "off8"])
@pytest.mark.parametrize("k", [28, 29, 30])
def test_c2c_roundtrip_full_length(fctx, k, off):
    n = 1 << k
    g = torch.Generator(device="cuda").manual_seed(k + off)
    v = _view(n, off)
    v.copy_(torch.randn(n, dtype=torch.complex64, device="cuda", generator=g))
    x = v.clone()
    fctx.fft_c2c(v, n, 1, 1)
    fctx.fft_c2c(v, n, 1, -1)
    torch.cuda.synchronize()
    num, den = 0.0, 0.0
    chunk = 1 << 26
    for s in range(0, n, chunk):
        a, b = v[s:s + chunk].to(torch.complex128) / n, x[s:s + chunk].to(torch.complex128)
        num += float((a - b).abs().pow(2).sum())
        den += float(b.abs().pow(2).sum())
    err = np.sqrt(num / den)
    print(f"c2c round trip n=2^{k} +{off}: rel-L2 {err:.3e}")
    assert err < 2 * REL_L2


# ----------------------------------------------------------------------------- R2C in place
@pytest.mark.parametrize("off", [0, 8], ids=["off0", "off8"])
@pytest.mark.parametrize("k", list(range(1, 32)))
def test_r2c_inplace_vs_float64(fctx, k, off):
    n = 1 << k
    v = _view(n + 2, off, dtype=torch.float32)
    if k <= 28:
        g = torch.Generator(device="cuda").manual_seed(233 + k + off)
        x = torch.rand(n, device="cuda", generator=g) * 2 - 1
        v[:n] = x
        fctx.fft_r2c_inplace(v, n)
        truth = torch.fft.rfft(x.double())
        del x
        got = torch.view_as_complex(v.view(-1, 2))
        err = _dev_rel_l2(got, truth)
        emax = float((got.to(torch.complex128) - truth).abs().max() / truth.abs().max())
    else:
        bins, amps = _tone_plan(n, seed=k * 10 + off, lo=1, hi=n // 2)
        _tones(n, bins, amps, v[:n], real=True)
        fctx.fft_r2c_inplace(v, n)
        torch.cuda.synchronize()
        err, emax = _tone_errors(torch.view_as_complex(v.view(-1, 2)), bins, amps * n / 2)
    print(f"r2c n=2^{k} +{off}: rel-L2 {err:.3e}, max {emax:.3e}")
    assert err < REL_L2
    assert emax < _elem_bound(n)


def test_r2c_rejects_a_float_pointer_off_complex_alignment(fctx):
    v = _view(4096 + 2, 4, dtype=torch.float32)
    before = fctx.launch_count
    assert _err_code(lambda: fctx.fft_r2c_inplace(v, 4096)) == E_INVALID
    assert _err_code(lambda: fctx.fft_c2c(v.data_ptr(), 1024, 1, 1)) == E_INVALID
    assert _err_code(lambda: fctx.watfft_c2c_backward(v.data_ptr(), 1024, 1)) == E_INVALID
    assert fctx.launch_count == before


# ----------------------------------------------------------------------------- waterfall FFT at +8
@pytest.mark.parametrize("L,rows", [(1 << 13, 301), (1 << 14, 150)])
def test_watfft_unaligned_two_sweep(fctx, L, rows):
    x = _uniform((rows, L), seed=L + rows)
    v = _view(rows * L, 8)
    v.copy_(x.reshape(-1))
    fctx.watfft_c2c_backward(v, L, rows)
    truth = torch.fft.ifft(x.to(torch.complex128), dim=-1, norm="forward")
    err = _dev_rel_l2(v.view(rows, L), truth)
    print(f"watfft +8 L=2^{L.bit_length() - 1} rows={rows}: rel-L2 {err:.3e}")
    assert err < REL_L2


# ----------------------------------------------------------------------------- element-wise stages at +8
def _at8(a):
    """device copy of complex64 numpy data at an address 8 bytes past 16-byte alignment"""
    v = _view(a.size, 8)
    v.copy_(torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda())
    return v


@pytest.mark.parametrize("nc", [(1 << 16) + 1, 1 << 16, 1001])
def test_rfi_s1_unaligned(fctx, oracle, nc):
    rng = np.random.default_rng(nc + 8)
    x = _spectrum(rng, nc, rng.integers(0, nc, 20))
    thr, C_ = 1.5, 16
    coef = srtb_b200.norm_coefficient(nc, C_)
    ranges = [(3, 17), (nc - 5, nc - 1)]
    ey, emean, emask = oracle.rfi_s1_average(x, thr, C_)
    for lo, hi in ranges:
        ey[lo:hi + 1] = 0
    means, outs = [], []
    for d in (_at8(x), torch.from_numpy(x).cuda()):
        dmean = torch.zeros(1, dtype=torch.float32, device="cuda")
        fctx.rfi_s1(d, nc, thr, coef, ranges, dmean)
        means.append(float(dmean.cpu()[0]))
        outs.append(d.cpu().numpy())
    got, aligned = outs
    truth_mean = float(np.mean(np.abs(x.astype(np.complex128)) ** 2))
    assert abs(means[0] - truth_mean) / truth_mean < 1e-6
    assert abs(means[0] - means[1]) / means[1] < 1e-6        # the 8-byte loop may reassociate the sum
    p = np.abs(x.astype(np.complex128)) ** 2
    border = np.abs(p / (thr * truth_mean) - 1) < BORDER
    for lo, hi in ranges:
        assert not got[lo:hi + 1].any()
    gmask = (got == 0) & (x != 0)
    emask = emask.astype(bool)
    for lo, hi in ranges:
        emask[lo:hi + 1] = True
    assert np.array_equal(gmask[~border], emask[~border])
    keep = ~gmask & ~emask
    assert rel_l2(got[keep], ey[keep]) < 1e-6
    assert rel_l2(got[keep], x[keep].astype(np.complex128) * coef) < 1e-6
    assert np.array_equal(got[~border], aligned[~border])


@pytest.mark.parametrize("nc", [(1 << 16) + 1, 1 << 14])
def test_dedisperse_unaligned(fctx, oracle, nc):
    rng = np.random.default_rng(nc + 9)
    x = (rng.standard_normal(nc) + 1j * rng.standard_normal(nc)).astype(np.complex64)
    f_min, bw, dm = np.float32(1000.0), np.float32(400.0), 562.05
    f_c = np.float32(f_min + bw)
    df = np.float32(bw / np.float32(nc))
    d = _at8(x)
    fctx.dedisperse(d, nc, float(f_min), float(f_c), float(df), dm)
    got = d.cpu().numpy()
    a = torch.from_numpy(x).cuda()
    fctx.dedisperse(a, nc, float(f_min), float(f_c), float(df), dm)
    expect = oracle.dedisperse(x, float(f_min), float(f_c), float(df), dm)
    i = np.arange(nc, dtype=np.longdouble)
    f = np.longdouble(f_min) + np.longdouble(df) * i
    k = np.longdouble(4.148808e3) * 1e6 * np.longdouble(np.float32(dm)) / f * ((f - np.longdouble(f_c)) / np.longdouble(f_c)) ** 2
    truth = x.astype(np.complex128) * np.exp(-2j * np.pi * (k - np.trunc(k)).astype(np.float64))
    tol = max(REL_L2, 2 * np.pi * float(np.abs(k).max()) * 2.3e-16 * 4)
    print(f"dedisperse +8 n={nc}: rel-L2 {rel_l2(got, truth):.3e}")
    assert rel_l2(got, truth) < tol
    assert rel_l2(got, expect) < 2 * tol
    assert rel_l2(got, a.cpu().numpy()) < 1e-6


@pytest.mark.parametrize("C_,L", [(64, 2048), (33, 1001)])
def test_rfi_s2_sk_unaligned(fctx, oracle, C_, L):
    rng = np.random.default_rng(C_ * L + 21)
    x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    x[5, :] = 3
    x[9, ::8] *= 9
    x[11, :] = 0
    thr = 1.05
    ey, esk, ezap = oracle.rfi_s2(x.reshape(-1), L, C_, thr)
    sks, outs = [], []
    for d in (_at8(x), torch.from_numpy(x.reshape(-1)).cuda()):
        dsk = torch.zeros(C_, dtype=torch.float32, device="cuda")
        fctx.rfi_s2_sk(d, L, C_, thr, dsk)
        sks.append(dsk.cpu().numpy())
        outs.append(d.cpu().numpy().reshape(C_, L))
    sk, got = sks[0], outs[0]
    fin = np.isfinite(esk)
    assert np.array_equal(np.isnan(sk), np.isnan(esk))
    assert np.allclose(sk[fin], esk[fin], rtol=1e-5)
    assert np.allclose(sk[fin], sks[1][fin], rtol=1e-5)
    lo, hi = oracle.sk_thresholds(L, thr)
    border = np.zeros(C_, bool)
    border[fin] = (np.abs(esk[fin] / hi - 1) < BORDER) | (np.abs(esk[fin] / lo - 1) < BORDER)
    gzap = np.all(got == 0, axis=1) & ~np.all(x == 0, axis=1)
    assert np.array_equal(gzap[~border], ezap[~border].astype(bool))
    assert ezap[5] == 1 and ezap[9] == 1 and ezap[11] == 0
    same = gzap == ezap.astype(bool)
    assert np.array_equal(got[same], ey.reshape(C_, L)[same])
    assert np.array_equal(got[~border], outs[1][~border])


@pytest.mark.parametrize("C_,L,reserved,maxbox", [(16, 256, 0, 16), (33, 1001, 100, 1024)])
def test_signal_detect_unaligned(fctx, oracle, C_, L, reserved, maxbox):
    rng = np.random.default_rng(C_ * L + 3)
    x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    x[:, L // 3:L // 3 + 8] *= 10
    x[1, :] = 0
    snr, chan_thr = 6.0, 0.9
    eres, eseries = oracle.signal_detect(x.reshape(-1), L, C_, reserved, snr, chan_thr, maxbox)
    h = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
    res = fctx.signal_detect(_at8(x), L, C_, reserved, snr, chan_thr, maxbox, h, copy_all=True)
    _compare_detect(res, eres, h, eseries, snr)
    assert res.signal_count[0] > 0
    ha = np.zeros_like(h)
    ra = fctx.signal_detect(torch.from_numpy(x.reshape(-1)).cuda(), L, C_, reserved, snr, chan_thr, maxbox, ha,
                            copy_all=True)
    _compare_detect(res, ra, h, ha, snr)


def test_sk_v1_unaligned(fctx, oracle):
    nt, nf = 1000, 48
    x = _refft_layout_block(np.random.default_rng(nt + nf), nt, nf)
    thr = 1.1
    ey, esk, ezap = oracle.sk_v1(x.reshape(-1), nf, nt, thr)
    d = _at8(x)
    dsk = torch.zeros(nf, dtype=torch.float32, device="cuda")
    fctx.rfi_sk_v1(d, nf, nt, thr, dsk)
    got, sk = d.cpu().numpy().reshape(nt, nf), dsk.cpu().numpy()
    fin = np.isfinite(esk)
    assert np.array_equal(np.isnan(sk), np.isnan(esk))
    assert np.allclose(sk[fin], esk[fin], rtol=2e-5)
    lo, hi = oracle.sk_thresholds(nt, thr)
    border = np.zeros(nf, bool)
    border[fin] = (np.abs(esk[fin] / hi - 1) < BORDER) | (np.abs(esk[fin] / lo - 1) < BORDER)
    gzap = np.all(got == 0, axis=0) & ~np.all(x == 0, axis=0)
    assert np.array_equal(gzap[~border], ezap[~border].astype(bool))
    same = gzap == ezap.astype(bool)
    assert np.array_equal(got[:, same], ey.reshape(nt, nf)[:, same])


def test_signal_detect_v1_unaligned(fctx, oracle):
    nt, nf, maxbox = 1000, 48, 256
    x = _refft_layout_block(np.random.default_rng(7 * nt + nf), nt, nf)
    sk_thr, snr, chan_thr = 1.4, 5.0, 0.9
    espec, eres, eseries = oracle.signal_detect_v1(x.reshape(-1), nf, nt, sk_thr, snr, chan_thr, maxbox)
    d = _at8(x)
    h = np.zeros((srtb_b200.MAX_BOXCARS, nt), np.float32)
    res = fctx.signal_detect_v1(d, nf, nt, sk_thr, snr, chan_thr, maxbox, h, copy_all=True)
    assert np.array_equal(d.cpu().numpy().reshape(nt, nf), espec.reshape(nt, nf))
    _compare_detect(res, eres, h, eseries, snr)
    assert res.detect_enabled == 1 and res.signal_count[0] > 0


def test_elementwise_entries_reject_a_pointer_off_complex_alignment(fctx):
    buf = torch.zeros(4096, dtype=torch.float32, device="cuda")
    p = buf.data_ptr() + 4
    h = np.zeros((srtb_b200.MAX_BOXCARS, 64), np.float32)
    before = fctx.launch_count
    assert _err_code(lambda: fctx.rfi_s1(p, 64, 1.5, 1.0)) == E_INVALID
    assert _err_code(lambda: fctx.dedisperse(p, 64, 1000.0, 1500.0, 1.0, 10.0)) == E_INVALID
    assert _err_code(lambda: fctx.rfi_s2_sk(p, 64, 8, 1.1)) == E_INVALID
    assert _err_code(lambda: fctx.signal_detect(p, 64, 8, 0, 6.0, 0.9, 16, h)) == E_INVALID
    assert _err_code(lambda: fctx.rfi_sk_v1(p, 64, 8, 1.1)) == E_INVALID
    assert _err_code(lambda: fctx.signal_detect_v1(p, 8, 64, 1.1, 6.0, 0.9, 16, h)) == E_INVALID
    assert fctx.launch_count == before


def test_unpack_rejects_a_baseband_off_its_sample_width(fctx):
    """the one-stream unpack loads one sample at a time when a pointer is not 16-byte aligned: 16/32/64-bit samples
    need their natural alignment, and the float output 4 bytes"""
    d = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    out = torch.zeros(4096, dtype=torch.float32, device="cuda")
    p = d.data_ptr()
    before = fctx.launch_count
    for bits, off in [(16, 1), (-16, 1), (32, 2), (64, 4)]:
        assert _err_code(lambda: fctx.unpack(p + off, 16384, bits, srtb_b200.FORMAT_SIMPLE, 0, [out], 1024)) == E_INVALID
    assert _err_code(lambda: fctx.unpack(p + 1, 4096, 8, srtb_b200.FORMAT_SIMPLE, 0, [out.data_ptr() + 2], 1024)) == E_INVALID
    cfg = make_block_config(1 << 12, 16, srtb_b200.FORMAT_SIMPLE, 16, 0.0)
    assert _err_code(lambda: fctx.process_block(cfg, p + 1, 1 << 13, None, on_device=True)) == E_INVALID
    assert fctx.launch_count == before
    # the sample width is all they need: a 16-bit baseband at +2 bytes and an 8-bit one at +1 byte still unpack
    raw = np.random.default_rng(16).integers(0, 256, 4096, dtype=np.uint8)
    d[2:2 + raw.size] = torch.from_numpy(raw).cuda()
    fctx.unpack(p + 2, raw.size, 16, srtb_b200.FORMAT_SIMPLE, 0, [out], raw.size // 2)
    assert np.array_equal(out[:raw.size // 2].cpu().numpy(), raw.view(np.uint16).astype(np.float32))
    d[1:1 + raw.size] = torch.from_numpy(raw).cuda()
    fctx.unpack(p + 1, raw.size, -8, srtb_b200.FORMAT_SIMPLE, 0, [out], raw.size)
    assert np.array_equal(out[:raw.size].cpu().numpy(), raw.view(np.int8).astype(np.float32))


# ----------------------------------------------------------------------------- block path
def _unpacked_2bit(raw):
    """unsigned 2-bit samples, MSB first (unpack.hpp:43-156)"""
    return np.stack([(raw >> s) & 3 for s in (6, 4, 2, 0)], axis=1).reshape(-1).astype(np.float64)


@pytest.mark.parametrize("bits", [-8, 2])
def test_block_unaligned_baseband(fctx, bits):
    n, C_ = 1 << 20, 64
    if bits == -8:
        bb = synth_baseband(n, seed=77, tone=False, pulse=True)
        raw, samples = bb.view(np.uint8), bb
    else:
        raw = np.random.default_rng(78).integers(0, 256, n // 4, dtype=np.uint8)
        samples = _unpacked_2bit(raw)
    cfg = make_block_config(n, bits, srtb_b200.FORMAT_SIMPLE, C_, 56.778, avg_thr=1e9, sk_thr=1.95, snr=6.0)
    d = torch.zeros(raw.size + 16, dtype=torch.uint8, device="cuda")
    d[1:1 + raw.size] = torch.from_numpy(raw).cuda()
    res = fctx.process_block(cfg, d.data_ptr() + 1, raw.size, None, on_device=True)
    L = n // 2 // C_
    got = _from_device_ptr(fctx.block_spectrum_ptr(0), n // 2).reshape(C_, L)
    truth = chain_truth_float64(samples, cfg)
    # SK may zap a channel (the unsigned 2-bit samples put their DC level into channel 0): compare the kept ones
    keep = ~np.all(got == 0, axis=1)
    assert keep.sum() >= C_ - 1
    err = rel_l2(got[keep], truth[keep])
    print(f"block +1 byte, bits {bits}: rel-L2 {err:.3e} over {int(keep.sum())} of {C_} channels")
    assert err < REL_L2
    d[:raw.size] = torch.from_numpy(raw).cuda()
    ra = fctx.process_block(cfg, d, raw.size, None, on_device=True)
    assert res[0].zero_count == ra[0].zero_count and res[0].n_boxcars == ra[0].n_boxcars
    assert res[0].detect_enabled == ra[0].detect_enabled
    for b in range(res[0].n_boxcars):
        assert res[0].threshold[b] == pytest.approx(ra[0].threshold[b], rel=1e-4)
        assert abs(int(res[0].signal_count[b]) - int(ra[0].signal_count[b])) <= 2


def test_block_two_stream_format_needs_aligned_baseband(fctx):
    n = 1 << 20
    d = torch.zeros(2 * n + 16, dtype=torch.uint8, device="cuda")
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, 64, 0.0)
    before = fctx.launch_count
    assert _err_code(lambda: fctx.process_block(cfg, d.data_ptr() + 1, 2 * n, None, on_device=True)) == E_INVALID
    assert fctx.launch_count == before


def test_submit_block_rejects_unaligned_spectrum_buffer(fctx):
    n = 1 << 16
    bb = torch.from_numpy(synth_baseband(n, seed=5).view(np.uint8).copy()).cuda()
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, 16, 0.0)
    spec = torch.zeros(n + 8, dtype=torch.float32, device="cuda")
    before = fctx.launch_count
    assert _err_code(lambda: fctx.submit_block_ex(cfg, bb, n, on_device=True, d_spectrum=[spec.data_ptr() + 8])) == E_INVALID
    assert fctx.launch_count == before
    t = fctx.submit_block_ex(cfg, bb, n, on_device=True, d_spectrum=[spec])   # the ring is still usable
    assert len(fctx.collect_block(t)) == 1


# block-path routes (SK / chirp / raw first sweep variants), for kernel coverage: the chirp geometries of
# test_chirp_newton.GPU_CASES, and four that reach the remaining whole-row reciprocal variants in the DM sweep
# (test_chirp_newton.chirp_variant), through the block path and the DM sweep; one block per raw-byte format and
# first-sweep length
ROUTE_CASES = GPU_CASES + [
    ("sweep_bigrow_v1_16384", 1 << 24, 512, 1000.0, 0.05, 500.0),
    ("sweep_bigrow_v2_16384", 1 << 20, 32, 1000.0, 500.0, 0.02),
    ("sweep_bigrow_v4_16384", 1 << 20, 32, 1000.0, 64.0, 0.02),
    ("sweep_bigrow_v3_8192", 1 << 20, 64, 1000.0, 0.2, 0.02),
]


@pytest.mark.parametrize("case", ROUTE_CASES, ids=[c[0] for c in ROUTE_CASES])
def test_block_route(fctx, case):
    _, n, C_, f_low, bw, dm = case
    bb = synth_baseband(n, seed=n // C_, tone=False, pulse=False)
    cfg = make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                            avg_thr=1e9, sk_thr=1.95, snr=50.0)
    d = torch.from_numpy(bb.view(np.uint8).copy()).cuda()
    res = fctx.process_block(cfg, d, n, None, on_device=True)
    samples = torch.from_numpy(bb).cuda()
    _spectrum_vs_truth(f"{case[0]} block", fctx.block_spectrum_ptr(0), _chain_truth_dev(samples, cfg, dm))
    sweep = fctx.process_block_dm_sweep(cfg, d, n, [dm, dm / 2], on_device=True)
    _spectrum_vs_truth(f"{case[0]} sweep, last trial", fctx.sweep_spectrum_ptr(), _chain_truth_dev(samples, cfg, dm / 2))
    assert len(res) == 1 and res[0].zero_count == 0
    assert sweep[0][0].zero_count == 0 and sweep[0][0].n_boxcars == res[0].n_boxcars


@pytest.mark.parametrize("fmt,bits,logn", [
    ("SIMPLE", 8, 22), ("SIMPLE", 2, 22), ("SIMPLE", 4, 22), ("NAOCPSR_SNAP1", -8, 22), ("INTERLEAVED_2", 8, 22),
    ("GZNUPSR_A1_2", 8, 22),                                            # first sweep 2^7
    ("SIMPLE", 8, 23), ("SIMPLE", 4, 23),                               # 2^8
    ("SIMPLE", 8, 26), ("NAOCPSR_SNAP1", -8, 26),                       # 2^9
    ("SIMPLE", 8, 28), ("SIMPLE", 2, 28), ("NAOCPSR_SNAP1", -8, 28)])   # 2^7, 32 columns wide (four sweeps)
def test_block_raw_format(fctx, oracle, fmt, bits, logn):
    """the unpack fused into the first sweep, per raw-byte variant: every stream's dynamic spectrum against float64 of
    the samples the CPU oracle unpacks (thresholds out of the way, so no decision enters the comparison)"""
    n, C_, dm = 1 << logn, 64, 10.0
    streams = 1 if fmt == "SIMPLE" else 2
    nbytes = n * streams * abs(bits) // 8
    raw = np.random.default_rng(n + bits).integers(0, 256, nbytes, dtype=np.uint8)
    cfg = make_block_config(n, bits, getattr(srtb_b200, "FORMAT_" + fmt), C_, dm, avg_thr=1e9, sk_thr=1.95, snr=50.0)
    res = fctx.process_block(cfg, torch.from_numpy(raw).cuda(), nbytes, None, on_device=True)
    assert len(res) == streams
    if fmt == "SIMPLE":
        samples = [oracle.unpack(raw, n, bits)]
    elif fmt == "NAOCPSR_SNAP1":
        samples = oracle.unpack_snap1(raw, n)
    elif fmt == "INTERLEAVED_2":
        samples = oracle.unpack_interleaved_2(raw, n, bits)
    else:
        samples = oracle.unpack_gznupsr_a1(raw, n, 2)
    for s in range(streams):
        truth = _chain_truth_dev(torch.from_numpy(samples[s]).cuda(), cfg, dm)
        _spectrum_vs_truth(f"raw {fmt} {bits}-bit 2^{logn}, stream {s}", fctx.block_spectrum_ptr(s), truth)
        del truth


# ----------------------------------------------------------------------------- size errors (host side)
def test_fft_size_and_argument_errors(fctx):
    d = torch.zeros(4096, dtype=torch.complex64, device="cuda")
    before = fctx.launch_count
    assert _err_code(lambda: fctx.fft_c2c(d, 1 << 10, (1 << 24) + 1, 1)) == E_SIZE          # batch * n > 2^34
    assert _err_code(lambda: fctx.fft_c2c(d, 1 << 2, (1 << 32) + 1, 1)) == E_SIZE
    assert _err_code(lambda: fctx.fft_c2c(d, 1 << 31, 1, -1)) == E_SIZE                     # length above 2^30
    assert _err_code(lambda: fctx.watfft_c2c_backward(d, 1 << 31, 1)) == E_SIZE
    assert _err_code(lambda: fctx.fft_r2c_inplace(d, 1 << 32)) == E_SIZE                     # n_real above 2^31
    assert _err_code(lambda: fctx.fft_c2c(None, 1024, 1, 1)) == E_INVALID
    assert _err_code(lambda: fctx.fft_c2c(d, 0, 1, 1)) == E_INVALID
    assert _err_code(lambda: fctx.fft_c2c(d, 1024, 0, 1)) == E_INVALID
    assert _err_code(lambda: fctx.fft_r2c_inplace(None, 1024)) == E_INVALID
    assert _err_code(lambda: fctx.fft_r2c_inplace(d, 0)) == E_SIZE
    assert fctx.launch_count == before


# ----------------------------------------------------------------------------- kernel coverage
def test_every_listed_kernel_was_launched(request):
    """every FFT-engine kernel that the coverage table assigns to a case of this module ran in that case"""
    if not request.config.getoption("keyword"):   # every case of the module was collected: the table's ids exist
        here = {i.name for i in request.session.items if i.module is request.module}
        unknown = sorted({c for c in KERNEL_CASES.values() if not c.startswith("unreached:")} - here)
        assert not unknown, f"the coverage table names cases this module does not have: {unknown}"
    if not LAUNCHED:
        pytest.skip("no case of this module ran")
    if not any(PROFILER_SEES_KERNELS):
        pytest.skip("torch.profiler recorded no CUDA kernel at all, not even torch's own")
    missing = []
    for kern, case in KERNEL_CASES.items():
        if case.startswith("unreached:") or case not in LAUNCHED:
            continue   # deselected, or failed before its kernels were recorded
        if kern not in LAUNCHED[case]:
            missing.append(f"{kern} not launched by {case}")
    assert not missing, "\n".join(missing)
