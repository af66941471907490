#!/usr/bin/env python
"""Cost of the total-intensity detector (block config field signal_detect_sum_streams) at config #3: dual-polarisation
naocpsr_snap1 blocks of 2^26 8-bit samples per stream, C = 2^11 channels of L = 2^14, device-resident, through
srtb_b200_submit_block_device / collect_block (two blocks in flight).

Timed run: --rounds rounds, each of --blocks blocks with the sum off and then on (alternating in one process), a host
clock around each round that ends in the last collect; ms per block is the median over rounds, and the overhead is
on / off - 1. Profiled run (separate, after the timed one): torch.profiler over a few blocks with the sum on gives the
sum tail's own kernel time: stream_sum_mask_kernel + stream_sum_kernel + one colsum_final_scan_kernel + one
detect_boxcar_kernel (the mean duration of those two per launch, since the streams' detectors run them too).
The card's name and power limit are read in the same run. Prints one JSON line."""
import argparse
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
ap.add_argument("--blocks", type=int, default=20)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--out", default=None, help="directory for the profiler's kernel table (optional)")
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
n = 1 << 26
cfg = srtb_b200.BlockConfig()
cfg.baseband_input_count, cfg.baseband_input_bits = n, -8
cfg.baseband_format, cfg.window, cfg.baseband_reserve_sample = srtb_b200.FORMAT_NAOCPSR_SNAP1, 0, 0
cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = 1000.0, 400.0, 8e8, 562.05
cfg.mitigate_rfi_average_method_threshold, cfg.mitigate_rfi_spectral_kurtosis_threshold = 1.5, 1.05
cfg.spectrum_channel_count = 1 << 11
cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold = 8.0, 0.9
cfg.signal_detect_max_boxcar_length = 256
g = torch.Generator(device="cuda").manual_seed(0)
d_bb = (torch.randn(2 * n, device="cuda", generator=g) * 20).round().clamp(-127, 127).to(torch.int8)
nbytes = 2 * n


def run(sum_, blocks):
    cfg.signal_detect_sum_streams = sum_
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tickets = []
    for _ in range(blocks):
        tickets.append(ctx.submit_block_device(cfg, d_bb, nbytes))
        if len(tickets) == 2:
            ctx.collect_block(tickets.pop(0))
    for t in tickets:
        ctx.collect_block(t)
    return (time.perf_counter() - t0) / blocks * 1e3


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
for s in (0, 1):
    run(s, 3)  # warm-up: allocations, tables, both routes
ms = {0: [], 1: []}
for _ in range(args.rounds):
    for s in (0, 1):
        ms[s].append(run(s, args.blocks))
off, on = float(np.median(ms[0])), float(np.median(ms[1]))

launches0 = ctx.launch_count
run(0, 1)
per_block_off = ctx.launch_count - launches0
launches0 = ctx.launch_count
run(1, 1)
per_block_on = ctx.launch_count - launches0

from torch.profiler import ProfilerActivity, profile  # noqa: E402

prof_blocks = 5
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run(1, prof_blocks)
kern = {}
for e in prof.events():
    if e.device_type.name != "CUDA":
        continue
    k = kern.setdefault(e.name, [0, 0.0])
    k[0] += 1
    k[1] += e.device_time_range.elapsed_us() if hasattr(e, "device_time_range") else e.cuda_time_total


def mean_us(pattern):
    hits = [(c, t) for name, (c, t) in kern.items() if pattern in name]
    c = sum(h[0] for h in hits)
    return (sum(h[1] for h in hits) / c) if c else 0.0


def total_us(pattern):
    return sum(t for name, (c, t) in kern.items() if pattern in name) / prof_blocks


tail_us = (total_us("stream_sum_mask_kernel") + total_us("stream_sum_kernel") + mean_us("colsum_final_scan_kernel") +
           mean_us("detect_boxcar_kernel"))
if args.out:
    Path(args.out).mkdir(parents=True, exist_ok=True)
    (Path(args.out) / "stream_sum_kernels.txt").write_text(
        prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))
print(json.dumps({
    "card": card, "samples_per_stream": n, "streams": 2, "blocks_per_round": args.blocks, "rounds": args.rounds,
    "ms_per_block_off": round(off, 4), "ms_per_block_on": round(on, 4),
    "ms_per_block_off_all": [round(v, 4) for v in ms[0]], "ms_per_block_on_all": [round(v, 4) for v in ms[1]],
    "overhead": round(on / off - 1.0, 5), "launches_per_block_off": per_block_off,
    "launches_per_block_on": per_block_on,
    "sum_tail_kernel_us": round(tail_us, 2),
    "stream_sum_mask_kernel_us": round(total_us("stream_sum_mask_kernel"), 2),
    "stream_sum_kernel_us": round(total_us("stream_sum_kernel"), 2)}))
ctx.close()
