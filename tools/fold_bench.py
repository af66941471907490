#!/usr/bin/env python
"""Times srtb_b200_fold at the config #3 stream shape: 2 streams of 2^26 samples, C = 2^11 channels of L = 2^14,
random dynamic spectra already on the device, nsub in {1, 64, 2048} and nbin in {64, 1024}. CUDA events around each
call (the call synchronises once, after copying the profile to pinned host memory), 3 warm-up calls, the median of
--reps (default 10). Per case: ms per call, the bytes the fold must read (2 C L 8) over that time, and its share of the
H100 SXM data-sheet 3.35 TB/s; the profile's own bytes are listed beside them. Then a torch.profiler pass gives each
case's kernel time alone.

Then the per-block cost of folding on the executable's path: config #3 blocks (naocpsr_snap1, 8-bit, device-resident)
through submit_block_ex / collect_block_ex with two blocks in flight, with and without srtb_b200_fold on each collected
block's spectra (nsub 1, nbin 256, as baseband_chain_pipe calls it), alternating over --rounds rounds of --blocks blocks;
a host clock around each round. The card's name and power limit are read in the same run. Prints one JSON line.

With --coherence the same cases time srtb_b200_fold_coherence of the two streams instead (the same bytes read), and the
block path alternates three arms: no fold, srtb_b200_fold, and srtb_b200_fold followed by srtb_b200_fold_coherence, as
baseband_chain_pipe calls them with fold_coherence = 1."""
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
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
import srtb_b200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--blocks", type=int, default=20)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--coherence", action="store_true", help="time srtb_b200_fold_coherence of the stream pair")
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
n, C_ = 1 << 26, 1 << 11
L = n // 2 // C_
S = 2
g = torch.Generator(device="cuda").manual_seed(0)
xs = [torch.randn((C_, L, 2), device="cuda", generator=g, dtype=torch.float32) for _ in range(S)]
xs[0][7].zero_()
phase = srtb_b200.fold_phase(0.0893, 1.25e-13, 8e8, 2 * C_, 123456789)
PEAK = 3.35e12



def call(nsub, nbin):
    """(entry, its arguments, profile elements) of one case; pinned host outputs: at nsub = 2048 the profile is 32 MiB
    (64 MiB for the coherence products), and its copy to pageable memory would dominate"""
    P = 4 if args.coherence else S
    prof = torch.zeros(P * nsub * nbin, dtype=torch.float64).pin_memory()
    hits = torch.zeros(nbin, dtype=torch.int64).pin_memory()
    kept = torch.zeros(P * nsub, dtype=torch.int32).pin_memory()
    keep.append((prof, hits, kept))
    outs = (prof.data_ptr(), hits.data_ptr(), kept.data_ptr())
    if args.coherence:
        return (ctx.lib.srtb_b200_fold_coherence,
                (ctx.h, xs[0].data_ptr(), xs[1].data_ptr(), L, C_, L, *phase, nbin, nsub, *outs), P * nsub * nbin)
    arr = (C.c_void_p * S)(*[x.data_ptr() for x in xs])
    keep.append(arr)
    return ctx.lib.srtb_b200_fold, (ctx.h, arr, S, L, C_, L, *phase, nbin, nsub, *outs), P * nsub * nbin


keep = []  # the host outputs and pointer arrays of the calls
cases = []
for nsub in (1, 64, 2048):
    for nbin in (64, 1024):
        fn, args_, out_elems = call(nsub, nbin)
        for _ in range(3):
            assert fn(*args_) == 0
        l0 = ctx.launch_count
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args_)
            e1.record()
            assert rc == 0, rc
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        nbytes = S * C_ * L * 8
        cases.append({"nsub": nsub, "nbin": nbin, "ms_per_call": ms, "ms_all": times, "bytes": nbytes,
                      "output_bytes_copied_to_host": out_elems * 8,
                      "gb_per_s": nbytes / (ms * 1e-3) / 1e9, "share_of_3_35_tb_s": nbytes / (ms * 1e-3) / PEAK,
                      "launches_per_call": (ctx.launch_count - l0) / args.reps})

from torch.profiler import ProfilerActivity, profile  # noqa: E402

for case in cases:
    nsub, nbin = case["nsub"], case["nbin"]
    fn, args_, _ = call(nsub, nbin)
    with profile(activities=[ProfilerActivity.CUDA]) as pr:
        for _ in range(5):
            fn(*args_)
    us = 0.0
    for e in pr.events():
        if e.device_type.name == "CUDA" and "srtb_b200::fold" in e.name:
            us += e.device_time_range.elapsed_us() if hasattr(e, "device_time_range") else e.cuda_time_total
    case["kernel_ms_per_call"] = us / 5 / 1e3
    case["kernel_share_of_3_35_tb_s"] = case["bytes"] / (us / 5 * 1e-6) / PEAK if us else None

# ---- per block, the executable's path
cfg = srtb_b200.BlockConfig()
cfg.baseband_input_count, cfg.baseband_input_bits = n, -8
cfg.baseband_format, cfg.window, cfg.baseband_reserve_sample = srtb_b200.FORMAT_NAOCPSR_SNAP1, 0, 0
cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = 1000.0, 400.0, 8e8, 562.05
cfg.mitigate_rfi_average_method_threshold, cfg.mitigate_rfi_spectral_kurtosis_threshold = 1.5, 1.05
cfg.spectrum_channel_count = C_
cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold = 8.0, 0.9
cfg.signal_detect_max_boxcar_length = 256
d_bb = (torch.randn(2 * n, device="cuda", generator=g) * 20).round().clamp(-127, 127).to(torch.int8)
del xs
specs = [[torch.empty(n + 2, device="cuda") for _ in range(S)] for _ in range(3)]
h_series = [torch.zeros(S * srtb_b200.MAX_BOXCARS * L, dtype=torch.float32).pin_memory() for _ in range(3)]
NBIN = 256
fprof = np.zeros((S, 1, NBIN))
fhits = np.zeros(NBIN, np.uint64)
fkept = np.zeros((S, 1), np.uint32)
fcoh = np.zeros((4, 1, NBIN))
fckept = np.zeros(1, np.uint32)


def run(fold, blocks):
    """fold: 0 = none, 1 = srtb_b200_fold, 2 = srtb_b200_fold and srtb_b200_fold_coherence"""
    def collect(ticket):
        _, _, dspec = ctx.collect_block_ex(ticket)
        if fold:
            arr = (C.c_void_p * S)(*dspec[:S])
            assert ctx.lib.srtb_b200_fold(ctx.h, arr, S, L, C_, L, *phase, NBIN, 1, fprof.ctypes.data,
                                          fhits.ctypes.data, fkept.ctypes.data) == 0
        if fold == 2:
            assert ctx.lib.srtb_b200_fold_coherence(ctx.h, dspec[0], dspec[1], L, C_, L, *phase, NBIN, 1,
                                                    fcoh.ctypes.data, fhits.ctypes.data, fckept.ctypes.data) == 0

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tickets = []
    for b in range(blocks):
        tickets.append(ctx.submit_block_ex(cfg, d_bb, 2 * n, True, specs[b % 3], h_series[b % 3]))
        if len(tickets) == 2:
            collect(tickets.pop(0))
    for t in tickets:
        collect(t)
    return (time.perf_counter() - t0) / blocks * 1e3


arms = (0, 1, 2) if args.coherence else (0, 1)
for f in arms:
    run(f, 3)
ms = {f: [] for f in arms}
for _ in range(args.rounds):
    for f in arms:
        ms[f].append(run(f, args.blocks))
off, on = float(np.median(ms[0])), float(np.median(ms[1]))
block_path = {"blocks_per_round": args.blocks, "rounds": args.rounds, "fold_nsub": 1, "fold_nbin": NBIN,
              "ms_per_block_off": off, "ms_per_block_on": on, "overhead": on / off - 1,
              "ms_off_all": ms[0], "ms_on_all": ms[1]}
if args.coherence:
    coh = float(np.median(ms[2]))
    block_path.update({"ms_per_block_fold_and_coherence": coh, "coherence_ms_per_block": coh - on,
                       "ms_fold_and_coherence_all": ms[2]})
print(json.dumps({
    "workload": f"fold{' coherence' if args.coherence else ''}, config #3 stream shape: {S} streams of 2^26 samples, "
                f"C = {C_}, L = {L}",
    "card": card, "cases": cases, "block_path": block_path}))
ctx.close()
