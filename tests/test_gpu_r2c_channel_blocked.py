"""The config-#3 row sweep stores its spectrum channel-blocked (bin k1 + P k2 at (k2 >> 3) L + 8 k1 + (k2 & 7)) into the
stream's buffer, and the waterfall kernel transforms each channel there in place: manual zap ranges across channel and
k2' edges against float64, the ring with caller-owned buffers (which the row sweep now writes) against process_block,
and six launches per stream."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import srtb_b200  # noqa: E402
from test_gpu_parity import REL_L2, _from_device_ptr, chain_truth_float64, make_block_config, rel_l2  # noqa: E402
from test_gpu_r2c_sweep_order import BW, C_, DM, F_LOW, FS, L, N, P, _block  # noqa: E402

pytestmark = pytest.mark.gpu

NC = N // 2


def _freq(k):
    return F_LOW + BW * k / NC


# one range across the edge of channels 999 | 1000 (bin 1000 L), one across a k2' edge inside a channel
# (bin P (8 c + 3), c = 1100), one across both edges at once (bin 1500 L), in MHz around those bins
EDGES = [1000 * L, P * (8 * 1100 + 3), 1500 * L]
PAIRS = [(_freq(k - 40.5), _freq(k + 23.5)) for k in EDGES]


def _cfg(avg_thr=1e9, sk_thr=1.95, snr=50.0):
    return make_block_config(N, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, C_, DM, f_low=F_LOW, bw=BW, fs=FS, avg_thr=avg_thr,
                             sk_thr=sk_thr, snr=snr, maxbox=256, pairs=PAIRS)


def _zap_bins():
    out = []
    for lo_f, hi_f in PAIRS:
        lo_hi = srtb_b200.rfi_range_to_bins(lo_f, hi_f, F_LOW, BW, NC)
        assert lo_hi is not None
        out.append(tuple(lo_hi))
    return out


@pytest.fixture(scope="module")
def block():
    return _block(seed=4242)


def test_zap_across_channel_edges_vs_float64(ctx, block):
    """ranges that straddle channel and k2' edges: the dynamic spectrum within the float64 policy, every zapped bin
    zero in the frequency domain and its neighbours outside the range kept; six launches per stream"""
    raw, streams = block
    zb = _zap_bins()
    for (lo, hi), k in zip(zb, EDGES):
        assert lo < k <= hi, (lo, k, hi)   # the range covers both sides of the edge
    cfg = _cfg()
    pinned = torch.from_numpy(raw.view(np.uint8)).pin_memory()
    ctx.process_block(cfg, pinned, raw.size, None)
    torch.cuda.synchronize()
    l0 = ctx.launch_count
    ctx.process_block(cfg, pinned, raw.size, None)
    torch.cuda.synchronize()
    # per stream: raw column sweep, row sweep, one zap launch (up to 16 ranges), whole-row kernel, two detector kernels
    assert ctx.launch_count - l0 == 2 * 6
    for s in range(2):
        got = _from_device_ptr(ctx.block_spectrum_ptr(s), NC).reshape(C_, L)
        truth = chain_truth_float64(streams[s], cfg, zb)
        err = rel_l2(got, truth)
        rms = np.sqrt(np.mean(np.abs(truth) ** 2))
        assert err < REL_L2, (s, err)
        assert np.abs(got - truth).max() < 1e-4 * rms
        G = np.fft.fft(got.astype(np.complex128), axis=1).reshape(-1)
        T = np.fft.fft(truth, axis=1).reshape(-1)
        trms = np.sqrt(np.mean(np.abs(T) ** 2))
        for lo, hi in zb:
            assert np.abs(G[lo:hi + 1]).max() < 1e-4 * trms, (s, lo, hi)
            for k in (lo - 1, hi + 1):   # the first bins outside the range are not zapped
                assert abs(G[k] - T[k]) < 1e-3 * max(abs(T[k]), trms), (s, k)
                assert abs(T[k]) > 1e-3 * trms


def test_ring_with_caller_buffers_across_edges(ctx, block):
    """the ring, with caller-owned spectrum buffers that the row sweep writes into, leaves bit for bit what
    process_block leaves, zap ranges across the edges included"""
    raw, _ = block
    cfg = _cfg(avg_thr=1.5, sk_thr=1.05, snr=8.0)
    b = torch.from_numpy(raw.view(np.uint8)).pin_memory()
    expect = ctx.process_block(cfg, b, raw.size, None)
    torch.cuda.synchronize()
    espec = [_from_device_ptr(ctx.block_spectrum_ptr(s), NC) for s in range(2)]
    specs = [torch.full((N + 2,), float("nan"), dtype=torch.float32, device="cuda") for _ in range(2)]
    t = ctx.submit_block_ex(cfg, b, raw.size, False, specs, None)
    res, _, spec_ptrs = ctx.collect_block_ex(t)
    for s in range(2):
        assert int(spec_ptrs[s]) == specs[s].data_ptr()
        assert np.array_equal(_from_device_ptr(spec_ptrs[s], NC), espec[s]), f"stream {s}: spectrum differs"
        assert int(res[s].zero_count) == int(expect[s].zero_count)
        assert list(res[s].signal_count[:res[s].n_boxcars]) == list(expect[s].signal_count[:expect[s].n_boxcars])
