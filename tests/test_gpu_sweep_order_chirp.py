"""The chirp of the config-#3 sweep-order route (2 x 2^26 8-bit samples, C = 2^11, rows of 2^14): the whole-row
waterfall kernel evaluates every bin's phase in fp64 as it gathers a channel, with no phase table, so nothing is
rebuilt when the band or the DM changes. Against float64 (rel-L2 <= 1e-5 and max-abs <= 1e-4 RMS, the parity policy of
test_gpu_parity.py) with zapping off: an inverted band (df < 0), a large DM (|k| ~ 1e9 cycles, where a wrong
reciprocal or bin index shows), and DMs alternating between consecutive blocks of one context, through process_block
and the ring."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import srtb_b200  # noqa: E402
from test_gpu_parity import _from_device_ptr, chain_truth_float64, make_block_config, rel_l2, synth_baseband  # noqa: E402

pytestmark = pytest.mark.gpu

N = 1 << 26          # samples per stream: M = 2^25 complex points = 2^11 channels of 2^14
C_ = 1 << 11
L = N // 2 // C_
REL_L2 = 1e-5
MAX_ABS = 1e-4       # times the RMS of the float64 truth
LAUNCHES = 2 * 5     # per stream: two R2C sweeps, the waterfall kernel, two detector kernels (no manual zap range)


def _block(seed):
    """two int8 streams in the naocpsr_snap1 layout (re0 im0 re1 im1 per point), so the fused raw first sweep and the
    sweep-order route apply; noise only, so that no channel falls outside the wide SK window"""
    s = [synth_baseband(N, seed=seed + i, tone=False, pulse=False) for i in range(2)]
    raw = np.empty(2 * N, np.int8)
    v = raw.reshape(-1, 2, 2)
    v[:, 0, :] = s[0].reshape(-1, 2)
    v[:, 1, :] = s[1].reshape(-1, 2)
    return raw, s


def _cfg(dm, f_low=1000.0, bw=500.0):
    return make_block_config(N, -8, srtb_b200.FORMAT_NAOCPSR_SNAP1, C_, dm, f_low=f_low, bw=bw, fs=2e6 * abs(bw),
                             avg_thr=1e9, sk_thr=1.95, snr=50.0)


def _spectra(ptrs):
    torch.cuda.synchronize()
    return [_from_device_ptr(p, N // 2).reshape(C_, L) for p in ptrs]


def _check(label, got, truth):
    err = rel_l2(got, truth)
    rms = np.sqrt(np.mean(np.abs(truth) ** 2))
    mx = float(np.abs(got.astype(np.complex128) - truth).max() / rms)
    print(f"{label}: rel-L2 {err:.3e}, max-abs {mx:.3e} RMS")
    assert err <= REL_L2, f"{label}: rel-L2 {err:.3e}"
    assert mx <= MAX_ABS, f"{label}: max-abs {mx:.3e} RMS"


def _process(ctx, cfg, pinned, nbytes):
    """process_block on the sweep-order route (checked by its launch count); the streams' dynamic spectra"""
    l0 = ctx.launch_count
    res = ctx.process_block(cfg, pinned, nbytes, None)
    torch.cuda.synchronize()
    assert ctx.launch_count - l0 == LAUNCHES
    assert all(r.zero_count == 0 for r in res)
    return _spectra([ctx.block_spectrum_ptr(s) for s in range(2)])


@pytest.fixture(scope="module")
def block():
    raw, streams = _block(seed=4242)
    return raw, streams, torch.from_numpy(raw.view(np.uint8)).pin_memory()


@pytest.mark.parametrize("label,dm,f_low,bw", [("inverted band", 562.05, 1437.0, -400.0),
                                               ("large DM", 3000.0, 1000.0, 500.0)])
def test_sweep_order_chirp_vs_float64(ctx, block, label, dm, f_low, bw):
    raw, streams, pinned = block
    cfg = _cfg(dm, f_low, bw)
    got = _process(ctx, cfg, pinned, raw.size)
    for s in range(2):
        _check(f"{label}, stream {s}", got[s], chain_truth_float64(streams[s], cfg))


def test_alternating_dms_on_one_context(ctx, block):
    """DM a, b, a through process_block and then through the ring (all three blocks in flight at once, each with its
    own spectrum buffers): every spectrum matches float64 at its DM, the two DM-a blocks of each entry point are
    bit-identical to each other and to a fresh context's"""
    raw, streams, pinned = block
    dm_a, dm_b = 562.05, 1234.5
    dms = (dm_a, dm_b, dm_a)
    cfgs = [_cfg(d) for d in dms]
    got = [_process(ctx, c, pinned, raw.size) for c in cfgs]
    specs = [[torch.empty(N + 2, dtype=torch.float32, device="cuda") for _ in range(2)] for _ in dms]
    tickets = [ctx.submit_block_ex(c, pinned, raw.size, False, sp) for c, sp in zip(cfgs, specs)]
    ring = []
    for t in tickets:
        res, _, ptrs = ctx.collect_block_ex(t)
        assert all(r.zero_count == 0 for r in res)
        ring.append(_spectra(ptrs))
    fresh = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        first = _process(fresh, cfgs[0], pinned, raw.size)
    finally:
        fresh.close()
    for s in range(2):
        for d, i in ((dm_a, 0), (dm_b, 1)):
            truth = chain_truth_float64(streams[s], cfgs[i])
            _check(f"process_block DM {d}, stream {s}", got[i][s], truth)
            _check(f"ring DM {d}, stream {s}", ring[i][s], truth)
        for name, g in (("process_block", got), ("ring", ring)):
            assert np.array_equal(g[0][s], g[2][s]), f"{name}: the repeat at DM a differs, stream {s}"
            assert np.array_equal(g[0][s], first[s]), f"{name}: DM a differs from a fresh context's, stream {s}"
