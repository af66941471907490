"""Every chirp route and reciprocal variant of the waterfall, through both entry points (process_block and the DM
sweep), against float64.

The chirp is the one stage with a different implementation per route: a phase table or chirp_factor in the
sixteen-point row kernel, a table or Newton-step reciprocals in the whole-row kernel, Newton steps in the long-row
column sweep, dedisperse_kernel before a plain waterfall elsewhere. Which one runs follows from the geometry alone;
test_chirp_newton.py mirrors the host's selection, and the cases below are chosen with it so that every
(route, variant) is reached. Zapping is off in the value comparisons (s1 threshold 1e9, a wide SK window), so no
threshold decision enters them. Bounds: rel-L2 <= 1e-5 and max-abs <= 1e-4 RMS against float64 (the parity policy
of test_gpu_parity.py).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import srtb_b200  # noqa: E402
from test_chirp_newton import EXPECTED_PAIRS, GPU_CASES, ChirpParams, chirp_variant, gpu_case_pairs  # noqa: E402
from test_gpu_parity import _from_device_ptr, chain_truth_float64, make_block_config, rel_l2, synth_baseband  # noqa: E402

REL_L2 = 1e-5
MAX_ABS = 1e-4          # times the RMS of the float64 truth

assert gpu_case_pairs() == EXPECTED_PAIRS, "the cases no longer reach every (route, variant)"

CASES = {c[0]: c for c in GPU_CASES}
# the case whose manual-zap pair straddles the boundary between channel rows C/2 - 1 and C/2
ZAP_CASE = "long_n2_32768"


def _cfg(case, **kw):
    _, n, C_, f_low, bw, dm = case
    args = dict(f_low=f_low, bw=bw, fs=2e6 * abs(bw), avg_thr=1e9, sk_thr=1.95, snr=50.0)
    args.update(kw)
    return make_block_config(n, -8, srtb_b200.FORMAT_SIMPLE, C_, dm, **args)


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).pin_memory()


def _spectrum(ptr, C_, L):
    torch.cuda.synchronize()
    return _from_device_ptr(ptr, C_ * L).reshape(C_, L)


def _straddling_pair(case):
    """a manual-zap range (MHz) around the first bin of channel row C/2, and the bins it covers"""
    _, n, C_, f_low, bw, _ = case
    p = ChirpParams(*case[1:])
    edge = (C_ // 2) * p.L
    f_edge = p.f_min + p.df * edge
    pair = (f_edge - 40 * abs(p.df), f_edge + 40 * abs(p.df))
    bins = srtb_b200.rfi_range_to_bins(pair[0], pair[1], f_low, bw, n // 2)
    assert bins is not None and bins[0] < edge <= bins[1], (bins, edge)
    return pair, bins


def _check(label, got, truth):
    err = rel_l2(got, truth)
    rms = np.sqrt(np.mean(np.abs(truth) ** 2))
    mx = float(np.abs(got.astype(np.complex128) - truth).max() / rms)
    print(f"{label}: rel-L2 {err:.3e}, max-abs {mx:.3e} RMS")
    assert err <= REL_L2, f"{label}: rel-L2 {err:.3e}"
    assert mx <= MAX_ABS, f"{label}: max-abs {mx:.3e} RMS"


@pytest.mark.parametrize("name", list(CASES))
def test_chirp_route_vs_float64(ctx, name):
    """the dynamic spectrum of process_block and of a one-trial DM sweep at the same DM, against float64"""
    case = CASES[name]
    _, n, C_, f_low, bw, dm = case
    L = n // 2 // C_
    pairs, zap_bins = (), ()
    if name == ZAP_CASE:
        pair, bins = _straddling_pair(case)
        pairs, zap_bins = [pair], [bins]
    cfg = _cfg(case, pairs=pairs)
    bb = synth_baseband(n, seed=300 + list(CASES).index(name), tone=False, pulse=False)
    pinned = _pinned(bb)
    truth = chain_truth_float64(bb, cfg, zap_bins)
    block = ctx.process_block(cfg, pinned, n, None)[0]
    got_block = _spectrum(ctx.block_spectrum_ptr(0), C_, L)
    sweep = ctx.process_block_dm_sweep(cfg, pinned, n, [dm])[0][0]
    got_sweep = _spectrum(ctx.sweep_spectrum_ptr(), C_, L)
    for path, res, got in (("block", block, got_block), ("sweep", sweep, got_sweep)):
        route, variant = chirp_variant(n, C_, f_low, bw, dm, path)
        assert res.zero_count == 0
        _check(f"{name} {path}: {route} variant {variant}, L = {L}", got, truth)


def _header(r):
    return (int(r.zero_count), int(r.time_series_count), int(r.detect_enabled), int(r.n_boxcars),
            list(r.boxcar_length), list(r.series_length), list(r.signal_count), list(r.variance), list(r.threshold))


def _dispersed_pulse(n, f_low, bw, dm, seed, amp=200.0, width=48):
    """8-bit noise (sigma 20) plus a 48-sample burst dispersed at `dm` by the conjugate chirp in float64: the
    detector finds it at that DM, and a few channels fall outside the SK window"""
    rng = np.random.default_rng(seed)
    nc = n // 2
    pulse = np.zeros(n)
    pulse[n // 2:n // 2 + width] = rng.standard_normal(width) * amp
    X = np.fft.rfft(pulse)[:nc]
    f = f_low + (bw / nc) * np.arange(nc)
    f_c = f_low + bw
    k = 4.148808e3 * 1e6 * dm / f * ((f - f_c) / f_c) ** 2
    X *= np.exp(2j * np.pi * (k - np.trunc(k)))
    v = np.fft.irfft(np.concatenate([X, [0]]), n) + rng.standard_normal(n) * 20
    return np.clip(np.round(v), -127, 127).astype(np.int8)


def _snap1(a, b):
    raw = np.empty(2 * a.size, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = a.reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = b.reshape(-1, 2)
    return raw


@pytest.mark.parametrize("name,fmt", [("long_n2_32768", "simple"), ("long_n2_32768", "naocpsr_snap1"),
                                      ("long_n0_131072_inverted", "simple"), ("bigrow_v4_8192_inverted", "simple"),
                                      ("bigrow_v3_16384", "naocpsr_snap1"), ("row16_2048_inverted", "simple")])
def test_sweep_matches_block_path(ctx, name, fmt):
    """a block with a burst and a tone, real thresholds: every trial of a sweep gives what process_block gives at
    that DM. On the long route both entry points launch the same kernels with the same arguments into different
    buffers, so spectra and result headers are bit-identical; where the block path reads a phase table and the sweep
    evaluates the phase on the fly, thresholds agree within 1e-5 relative and signal counts within one."""
    case = CASES[name]
    _, n, C_, f_low, bw, dm = case
    L = n // 2 // C_
    streams = 2 if fmt == "naocpsr_snap1" else 1
    a = _dispersed_pulse(n, f_low, bw, dm, seed=500)
    raw = _snap1(a, _dispersed_pulse(n, f_low, bw, dm, seed=501)) if streams == 2 else a
    cfg = _cfg(case, avg_thr=5.0, sk_thr=1.3, snr=6.0, maxbox=256)
    cfg.baseband_format = srtb_b200.FORMAT_BY_NAME[fmt]
    pinned = _pinned(raw)
    exact = chirp_variant(n, C_, f_low, bw, dm, "block") == chirp_variant(n, C_, f_low, bw, dm, "sweep")
    dms = [0.0, dm] if dm != 0 else [dm]
    sweep = ctx.process_block_dm_sweep(cfg, pinned, raw.size, dms)
    last = _spectrum(ctx.sweep_spectrum_ptr(), C_, L)
    assert len(sweep) == len(dms) and all(len(r) == streams for r in sweep)
    for j, d in enumerate(dms):
        cfg.dm = d
        block = ctx.process_block(cfg, pinned, raw.size, None)
        assert len(block) == streams
        for s in range(streams):
            g, e = sweep[j][s], block[s]
            if exact:
                assert _header(g) == _header(e), f"DM {d} stream {s}"
            else:
                assert g.zero_count == e.zero_count and g.n_boxcars == e.n_boxcars
                for b in range(g.n_boxcars):
                    assert g.threshold[b] == pytest.approx(e.threshold[b], rel=1e-5)
                    assert abs(int(g.signal_count[b]) - int(e.signal_count[b])) <= 1
    for r in sweep[-1]:                                              # the pulse is found at its DM
        assert sum(int(c) for c in r.signal_count[:r.n_boxcars]) > 0
    spec = _spectrum(ctx.block_spectrum_ptr(streams - 1), C_, L)    # block path at the sweep's last DM
    if exact:
        assert np.array_equal(last, spec), "the sweep's last-trial spectrum differs from the block path's"
    else:
        same = np.all(last == 0, axis=1) == np.all(spec == 0, axis=1)
        assert same.all()
        assert rel_l2(last, spec) < 2 * REL_L2


@pytest.mark.parametrize("name", ["row16_1024", "bigrow_v3_16384", "bigrow_v4_8192_inverted", "long_n2_32768",
                                  "long_n1_32768", "unfused_512"])
def test_sweep_trial_does_not_depend_on_the_previous_one(ctx, name):
    """the last trial of a sweep over [dm_a, dm_b] equals a sweep over [dm_b] alone, bit for bit: a trial reads
    nothing the previous trial left in the sweep's buffers"""
    case = CASES[name]
    _, n, C_, _, _, dm = case
    L = n // 2 // C_
    cfg = _cfg(case, avg_thr=5.0, sk_thr=1.3, snr=6.0)
    pinned = _pinned(synth_baseband(n, seed=600))
    dm_a = -0.5 * dm if dm else 100.0
    two = ctx.process_block_dm_sweep(cfg, pinned, n, [dm_a, dm])
    got_two = _spectrum(ctx.sweep_spectrum_ptr(), C_, L)
    one = ctx.process_block_dm_sweep(cfg, pinned, n, [dm])
    got_one = _spectrum(ctx.sweep_spectrum_ptr(), C_, L)
    assert np.array_equal(got_two, got_one)
    assert _header(two[1][0]) == _header(one[0][0])


@pytest.mark.parametrize("name", ["row16_4096", "bigrow_v3_16384"])
def test_block_path_follows_the_dm_between_calls(ctx, name):
    """process_block at DM a, DM b, then a sweep, then DM a again: every spectrum matches float64 at its own DM (the
    phase table is rebuilt whenever the DM changes), and the repeat at DM a is bit-identical to the first"""
    case = CASES[name]
    _, n, C_, _, _, dm_a = case
    L = n // 2 // C_
    dm_b = 0.5 * dm_a
    bb = synth_baseband(n, seed=700, tone=False, pulse=False)
    pinned = _pinned(bb)
    cfg = _cfg(case)
    truth = {}
    for d in (dm_a, dm_b):
        cfg.dm = d
        truth[d] = chain_truth_float64(bb, cfg)
    got = []
    for step, d in enumerate((dm_a, dm_b, None, dm_a)):
        if d is None:
            ctx.process_block_dm_sweep(cfg, pinned, n, [dm_b, 2 * dm_a])
            continue
        cfg.dm = d
        res = ctx.process_block(cfg, pinned, n, None)[0]
        assert res.zero_count == 0
        got.append(_spectrum(ctx.block_spectrum_ptr(0), C_, L))
        _check(f"{name} call {step}: process_block at DM {d}", got[-1], truth[d])
    assert np.array_equal(got[0], got[2])
