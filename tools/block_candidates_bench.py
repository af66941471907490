#!/usr/bin/env python
"""Cost of listing the block path's single-pulse events (srtb_b200_submit_block_events) on the ring.

Config #3 (bench.py's "config3": 2^26 samples per stream, two streams, C = 2048, L = 16384, the sweep-order route),
device-resident: rounds of --blocks blocks through srtb_b200_submit_block_ex / collect_block_ex against the same blocks
through submit_block_events / collect_block_events (--max-events per detector), the two alternating round by round, the
ring kept full (SRTB_B200_RING_SLOTS in flight) as bench.py keeps it. ms per block is the median over --rounds of a
round's wall time (CUDA events) over its blocks. Two cases: noise at the configured S/N threshold 8 (few events), and a
busy threshold of 2.5 (thousands of events per block). With --sum, the total-intensity detector runs too. The events
pass's kernel time per block comes from torch.profiler over one round, and the launches from the ctx's counter. The card
and its power limit are read in the same run. Prints one JSON line."""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
import bench  # noqa: E402
import srtb_b200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--blocks", type=int, default=20)
ap.add_argument("--max-events", type=int, default=1 << 16)
ap.add_argument("--sum", action="store_true", help="also the total-intensity detector")
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
w = bench.WORKLOADS["config3"]
n, streams = 1 << w["log2n"], 2
cfg = srtb_b200.BlockConfig()
cfg.baseband_input_count, cfg.baseband_input_bits = n, w["bits"]
cfg.baseband_format, cfg.window, cfg.baseband_reserve_sample = srtb_b200.FORMAT_BY_NAME[w["fmt"]], 0, 0
cfg.baseband_freq_low, cfg.baseband_bandwidth = w["f_low"], w["bw"]
cfg.baseband_sample_rate, cfg.dm = w["fs"], w["dm"]
cfg.mitigate_rfi_average_method_threshold = w["avg_thr"]
cfg.mitigate_rfi_spectral_kurtosis_threshold = w["sk_thr"]
cfg.spectrum_channel_count = w["channels"]
cfg.signal_detect_channel_threshold = w["chan_thr"]
cfg.signal_detect_max_boxcar_length = w["maxbox"]
pairs = srtb_b200.eval_rfi_ranges(w["freq_list"])
flat = [v for p in pairs for v in p]
keep = (C.c_float * max(1, len(flat)))(*flat)
cfg.rfi_freq_pairs = C.cast(keep, C.POINTER(C.c_float))
cfg.n_rfi_freq_pairs = len(pairs)
cfg.signal_detect_sum_streams = 1 if args.sum else 0
blocks = [torch.from_numpy(bench.synth_block(n, streams, seed=i, bits=w["bits"]).view(np.uint8)).cuda()
          for i in range(4)]
torch.cuda.synchronize()
nbytes = blocks[0].numel()


def run_round(events: bool):
    """(wall ms per block, launches per block, events per block)"""
    pending, n_ev = [], 0
    l0 = ctx.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.blocks):
        if len(pending) == srtb_b200.RING_SLOTS:
            t = pending.pop(0)
            if events:
                out = ctx.collect_block_events(t)
                n_ev += sum(out[4]) + out[6]
            else:
                ctx.collect_block_ex(t)
        b = blocks[i % len(blocks)]
        pending.append(ctx.submit_block_events(cfg, b, nbytes, args.max_events, on_device=True) if events
                       else ctx.submit_block_ex(cfg, b, nbytes, on_device=True))
    for t in pending:
        if events:
            out = ctx.collect_block_events(t)
            n_ev += sum(out[4]) + out[6]
        else:
            ctx.collect_block_ex(t)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.blocks, (ctx.launch_count - l0) / args.blocks, n_ev / args.blocks


def events_kernel_us():
    """the two event kernels' device time per block, from torch.profiler over one round"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_round(True)
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if "ev_count_kernel" in e.key or "ev_emit_kernel" in e.key:
            tot += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return tot / args.blocks


cases = []
for snr in (w["snr"], 2.5):
    cfg.signal_detect_signal_noise_threshold = snr
    run_round(False)
    run_round(True)
    plain, evs = [], []
    for _ in range(args.rounds):
        plain.append(run_round(False))
        evs.append(run_round(True))
    p_ms = float(np.median([r[0] for r in plain]))
    e_ms = float(np.median([r[0] for r in evs]))
    cases.append(dict(snr=snr, plain_ms_per_block=round(p_ms, 4), events_ms_per_block=round(e_ms, 4),
                      overhead_pct=round(100.0 * (e_ms - p_ms) / p_ms, 2),
                      plain_launches_per_block=plain[0][1], events_launches_per_block=evs[0][1],
                      events_per_block=evs[0][2], events_kernels_us_per_block=round(events_kernel_us(), 2)))
print(json.dumps(dict(tool="block_candidates_bench", card=card, workload="config3", sum=bool(args.sum),
                      blocks=args.blocks, rounds=args.rounds, max_events=args.max_events, cases=cases)))
