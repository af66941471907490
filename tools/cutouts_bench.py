#!/usr/bin/env python
"""Cost of the candidate cut-outs (srtb_b200_candidate_cutouts) at the config #3 stream shape.

One stream's [C][L] spectrum (C = 2048, L = 16384, the last 1024 samples reserved), W = n_rows = 256, nsub = 256, the
executable's half-width rule ((W/2) q / max |k|). For q = 1, 16, 128 and n = 1, 8, 64 requests: ms per call (CUDA
events around the synchronising call, median over --rounds, the nine cases alternating call by call), ms per
candidate, and the plane's adds (W n_rows C per candidate) per second. The four kernels' device time per candidate comes
from torch.profiler in a separate pass. Then what one cut-out call adds to a config #3 block as the executable runs it
with candidate_cutouts = 8: the block's ms through the ring (submit_block_ex / collect_block_ex, device-resident, the
ring full) against the same rounds followed by one N = 8 call per stream (q = 1 .. 16), alternating round by round. The
card and its power limit are read in the same run. Prints one JSON line."""
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
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402
import cutout_oracle as co  # noqa: E402
import srtb_b200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=15)
ap.add_argument("--blocks", type=int, default=20)
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
w = bench.WORKLOADS["config3"]
Cn, L, R, W, ROWS, NSUB = 2048, 16384, 1024, 256, 256, 256
fl, bw, fs, dm = w["f_low"], w["bw"], w["fs"], w["dm"]
k_max = float(np.abs(co.k_table(Cn, fl, bw, fs)).max())
rng = np.random.default_rng(0)
x = (rng.standard_normal((Cn, L)) + 1j * rng.standard_normal((Cn, L))).astype(np.complex64)
d_x = torch.from_numpy(x.view(np.float32)).cuda()
ts = L - R


def requests(n, q, seed=1):
    r = np.random.default_rng(seed)
    hw = (W // 2) * q / k_max
    return [(int(r.integers(0, ts)), dm, hw, q) for _ in range(n)]


def call(reqs, spectra=None):
    return ctx.candidate_cutouts(spectra or [d_x], L, Cn, R, fl, bw, fs, dm, reqs, W, NSUB, ROWS)


def timed(reqs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call(reqs)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


cases = [(q, n) for q in (1, 16, 128) for n in (1, 8, 64)]
reqs = {c: requests(c[1], c[0]) for c in cases}
for c in cases:
    timed(reqs[c])
times = {c: [] for c in cases}
for _ in range(args.rounds):
    for c in cases:
        times[c].append(timed(reqs[c]))

# kernel time per candidate: the four cut-out kernels' device time, torch.profiler, one call per case
from torch.profiler import ProfilerActivity, profile  # noqa: E402

kern_us = {}
for c in cases:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(reqs[c])
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if "cutout_" in e.key:
            tot += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    kern_us[c] = tot

out_cases = []
for (q, n) in cases:
    ms = float(np.median(times[(q, n)]))
    adds = float(n) * W * ROWS * Cn
    out_cases.append(dict(q=q, n=n, ms_per_call=round(ms, 4), ms_per_candidate=round(ms / n, 4),
                          kernel_us_per_candidate=round(kern_us[(q, n)] / n, 2),
                          plane_adds_per_s_call=float(f"{adds / (ms * 1e-3):.3g}"),
                          plane_adds_per_s_kernels=float(f"{adds / (kern_us[(q, n)] * 1e-6):.3g}")))

# the executable's path: a config #3 block through the ring, with and without one N = 8 call per stream
n, streams = 1 << w["log2n"], 2
cfg = srtb_b200.BlockConfig()
cfg.baseband_input_count, cfg.baseband_input_bits = n, w["bits"]
cfg.baseband_format, cfg.window, cfg.baseband_reserve_sample = srtb_b200.FORMAT_BY_NAME[w["fmt"]], 0, 0
cfg.baseband_freq_low, cfg.baseband_bandwidth = w["f_low"], w["bw"]
cfg.baseband_sample_rate, cfg.dm = w["fs"], w["dm"]
cfg.mitigate_rfi_average_method_threshold = w["avg_thr"]
cfg.mitigate_rfi_spectral_kurtosis_threshold = w["sk_thr"]
cfg.spectrum_channel_count = w["channels"]
cfg.signal_detect_signal_noise_threshold = w["snr"]
cfg.signal_detect_channel_threshold = w["chan_thr"]
cfg.signal_detect_max_boxcar_length = w["maxbox"]
pairs = srtb_b200.eval_rfi_ranges(w["freq_list"])
flat = [v for p in pairs for v in p]
keep = (C.c_float * max(1, len(flat)))(*flat)
cfg.rfi_freq_pairs = C.cast(keep, C.POINTER(C.c_float))
cfg.n_rfi_freq_pairs = len(pairs)
blocks = [torch.from_numpy(bench.synth_block(n, streams, seed=i, bits=w["bits"]).view(np.uint8)).cuda()
          for i in range(4)]
Lb = n // 2 // w["channels"]
torch.cuda.synchronize()
nbytes = blocks[0].numel()
block_reqs = [(int(rng.integers(0, Lb - 1024)), dm, (W // 2) * q / k_max, q) for q in (1, 1, 2, 2, 4, 8, 16, 16)]


def run_round(cut: bool):
    pending = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()

    def collect():
        _, _, sp = ctx.collect_block_ex(pending.pop(0))
        if cut:  # the executable's call per stream, on the block's own spectra
            for s in range(streams):
                ctx.candidate_cutouts([sp[s]], Lb, w["channels"], 1024, fl, bw, fs, dm, block_reqs, W, NSUB, ROWS)

    for i in range(args.blocks):
        if len(pending) == srtb_b200.RING_SLOTS:
            collect()
        pending.append(ctx.submit_block_ex(cfg, blocks[i % len(blocks)], nbytes, on_device=True))
    while pending:
        collect()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.blocks


run_round(False)
run_round(True)
plain, cut = [], []
for _ in range(max(3, args.rounds // 3)):
    plain.append(run_round(False))
    cut.append(run_round(True))
p_ms, c_ms = float(np.median(plain)), float(np.median(cut))
print(json.dumps(dict(tool="cutouts_bench", card=card, shape=dict(C=Cn, L=L, reserved=R, W=W, n_rows=ROWS, nsub=NSUB),
                      rounds=args.rounds, cases=out_cases,
                      block_path=dict(workload="config3", n_per_stream=8, blocks=args.blocks,
                                      plain_ms_per_block=round(p_ms, 4), cutouts_ms_per_block=round(c_ms, 4),
                                      overhead_pct=round(100.0 * (c_ms - p_ms) / p_ms, 2)))))
