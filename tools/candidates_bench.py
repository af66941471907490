#!/usr/bin/env python
"""Cost of listing a DM search's single-pulse events (csrc/events.cuh) and clustering them into candidates.

Incoherent search at the config #3 stream shape (C = 2048, L = 16384, max boxcar 256) for 64, 256 and 1024 trials over
dm +- 1: srtb_b200_incoherent_dm_search against srtb_b200_incoherent_dm_search_events, calls alternating, CUDA events
around each (both synchronise), median of --reps after 3 warm-up calls each. Two spectra: noise at S/N threshold 8 (few
events), and a busy one (the same noise at threshold 2.5: tens of thousands of events per call), so that the
compaction and the host clustering (srtb_b200_cluster_events, timed on its own with a host clock) run under load.
Coherent sweep at the config #4 shape (2^27 samples, 21 trials): srtb_b200_process_block_dm_sweep_ex against
srtb_b200_process_block_dm_sweep_events with the same outputs, alternating, host clock around each synchronous call.
The card and its power limit are read in the same run. Prints one JSON line."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
import bench  # noqa: E402
import srtb_b200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--trials", default="64,256,1024")
ap.add_argument("--max-events", type=int, default=1 << 18)
ap.add_argument("--no-sweep", action="store_true", help="skip the coherent sweep")
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
max_ev = args.max_events
EV = srtb_b200._dtype_of(srtb_b200.Event)


def median_ms(ts):
    return float(np.median(ts))


# ---- incoherent search
C_, L = 1 << 11, 1 << 14
f_low, bw, sr, dm = 1000.0, 500.0, 1e9, 100.0
g = torch.Generator(device="cuda").manual_seed(0)
x = torch.randn((C_, L, 2), device="cuda", generator=g, dtype=torch.float32)
x[7].zero_()
inc = []
for snr in (8.0, 2.5):
    for n_dm in [int(v) for v in args.trials.split(",")]:
        dms = list(dm + np.linspace(-1.0, 1.0, n_dm))
        arr = (C.c_float * n_dm)(*dms)
        res = (srtb_b200.DetectResult * n_dm)()
        peaks = (srtb_b200.Peak * n_dm)()
        best = C.c_int32()
        h_series = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
        ev = np.zeros(max_ev, EV)
        n_ev = C.c_uint64()

        def plain():
            return ctx.lib.srtb_b200_incoherent_dm_search(ctx.h, x.data_ptr(), L, C_, 0, f_low, bw, sr, dm, arr, n_dm,
                                                          snr, 0.9, 256, res, C.cast(peaks, C.c_void_p), C.byref(best),
                                                          h_series.ctypes.data)

        def events():
            return ctx.lib.srtb_b200_incoherent_dm_search_events(
                ctx.h, x.data_ptr(), L, C_, 0, f_low, bw, sr, dm, arr, n_dm, snr, 0.9, 256, res,
                C.cast(peaks, C.c_void_p), C.byref(best), h_series.ctypes.data, ev.ctypes.data, max_ev,
                C.byref(n_ev))

        for _ in range(3):
            assert plain() == 0 and events() == 0
        n0 = ctx.launch_count
        plain()
        n1 = ctx.launch_count
        events()
        n2 = ctx.launch_count
        tp, te = [], []
        for _ in range(args.reps):
            for fn, ts in ((plain, tp), (events, te)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                assert fn() == 0
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
        kept = ev[:min(n_ev.value, max_ev)]
        tc = []
        for _ in range(max(3, args.reps // 2)):
            t0 = time.perf_counter()
            cands, n_c = srtb_b200.cluster_events(kept, dms)
            tc.append(1e3 * (time.perf_counter() - t0))
        T = res[0].time_series_count
        inc.append({"n_dm": n_dm, "snr_threshold": snr, "T": T, "events": int(n_ev.value), "candidates": n_c,
                    "plain_ms": median_ms(tp), "events_ms": median_ms(te), "events_over_plain": median_ms(te) /
                    median_ms(tp), "cluster_ms_host": median_ms(tc), "plain_launches": n1 - n0,
                    "events_launches": n2 - n1,
                    # the boxcar series the event pass reads: trials x boxcars x T floats
                    "series_bytes": n_dm * res[0].n_boxcars * T * 4})
out = {"card": card, "incoherent": {"workload": f"config #3 stream shape: C = {C_}, L = {L}, max boxcar 256",
                                    "runs": inc}}

# ---- coherent sweep, config #4 shape
if not args.no_sweep:
    n = 1 << 27
    dms = [50.0 * i for i in range(21)]
    cfg = srtb_b200.BlockConfig()
    cfg.baseband_input_count, cfg.baseband_input_bits, cfg.baseband_format = n, -8, srtb_b200.FORMAT_SIMPLE
    cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = 1000.0, 500.0, 1e9, 0.0
    cfg.mitigate_rfi_average_method_threshold, cfg.mitigate_rfi_spectral_kurtosis_threshold = 5.0, 1.05
    cfg.spectrum_channel_count = 1 << 11
    cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold = 8.0, 0.9
    cfg.signal_detect_max_boxcar_length = 256
    blk = torch.from_numpy(bench.synth_block(n, 1, 4).view(np.uint8)).cuda()
    Lc = n // 2 // cfg.spectrum_channel_count
    # the C entries alone, with every buffer made beforehand (the Python wrappers allocate and convert per call)
    h_series = torch.zeros((1, srtb_b200.MAX_BOXCARS, Lc), dtype=torch.float32).pin_memory()
    d_spec = torch.empty(n + 2, dtype=torch.float32, device="cuda")
    arr = (C.c_float * len(dms))(*dms)
    res = (srtb_b200.DetectResult * len(dms))()
    peaks = (srtb_b200.Peak * len(dms))()
    best = (C.c_int32 * 4)()
    outs = srtb_b200.SweepOutputs()
    outs.h_peaks, outs.h_best_trial = C.cast(peaks, C.c_void_p), C.cast(best, C.c_void_p)
    outs.h_series = h_series.data_ptr()
    outs.d_spectrum[0] = d_spec.data_ptr()
    ev = np.zeros(max_ev, EV)
    n_ev = (C.c_uint64 * 4)()

    def ex():
        return ctx.lib.srtb_b200_process_block_dm_sweep_ex(ctx.h, C.byref(cfg), blk.data_ptr(), n, 1, arr, len(dms),
                                                           res, C.byref(outs))

    def events():
        return ctx.lib.srtb_b200_process_block_dm_sweep_events(ctx.h, C.byref(cfg), blk.data_ptr(), n, 1, arr,
                                                               len(dms), res, C.byref(outs), ev.ctypes.data, max_ev,
                                                               n_ev)

    for _ in range(2):
        assert ex() == 1 and events() == 1
    n0 = ctx.launch_count
    ex()
    n1 = ctx.launch_count
    events()
    n2 = ctx.launch_count
    tp, te = [], []
    for _ in range(args.reps):
        for fn, ts in ((ex, tp), (events, te)):
            t0 = time.perf_counter()
            assert fn() == 1
            ts.append(1e3 * (time.perf_counter() - t0))
    out["sweep"] = {"workload": f"config #4 shape: 2^27 samples x {len(dms)} trial DMs", "ex_ms": median_ms(tp),
                    "events_ms": median_ms(te), "events_over_ex": median_ms(te) / median_ms(tp),
                    "events": int(n_ev[0]), "ex_launches": n1 - n0, "events_launches": n2 - n1,
                    "ex_ms_all": tp, "events_ms_all": te}
print(json.dumps(out))
