#!/usr/bin/env python
"""BASELINE config #4 shape: one 2^27-sample 8-bit block swept over 21 trial DMs (0..1000, step 50) with
srtb_b200_process_block_dm_sweep (unpack + R2C once, then per DM: s1 + chirp + waterfall FFT + SK + detect).
Prints one JSON line: blocks/s, trial-Gsamples/s (samples x trials / time) and ms per trial.
--outputs: time the plain entry and srtb_b200_process_block_dm_sweep_ex with every output (peaks, best trial, the best
trial's series and spectrum) alternating in one run, and print both, their ratio and the card with its power limit."""
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

args = [a for a in sys.argv[1:] if a != "--outputs"]
with_outputs = "--outputs" in sys.argv[1:]
log2n = int(args[0]) if len(args) > 0 else 27
reps = int(args[1]) if len(args) > 1 else 5
n = 1 << log2n
dms = [50.0 * i for i in range(21)]
torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
cfg = srtb_b200.BlockConfig()
cfg.baseband_input_count, cfg.baseband_input_bits, cfg.baseband_format = n, -8, srtb_b200.FORMAT_SIMPLE
cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = 1000.0, 500.0, 1e9, 0.0
cfg.mitigate_rfi_average_method_threshold, cfg.mitigate_rfi_spectral_kurtosis_threshold = 5.0, 1.05
cfg.spectrum_channel_count = 1 << 11
cfg.signal_detect_signal_noise_threshold, cfg.signal_detect_channel_threshold = 8.0, 0.9
cfg.signal_detect_max_boxcar_length = 256
blk = torch.from_numpy(bench.synth_block(n, 1, 4).view(np.uint8)).cuda()
ctx.process_block_dm_sweep(cfg, blk, n, dms, on_device=True)
torch.cuda.synchronize()
if with_outputs:
    # both entries are synchronous: a host clock around each call times it whole
    L = n // 2 // cfg.spectrum_channel_count
    h_series = torch.zeros((1, srtb_b200.MAX_BOXCARS, L), dtype=torch.float32).pin_memory()
    d_spec = [torch.empty(n + 2, dtype=torch.float32, device="cuda")]
    ctx.process_block_dm_sweep(cfg, blk, n, dms, on_device=True, outputs=True, h_series=h_series, d_spectrum=d_spec)
    plain, ex = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ctx.process_block_dm_sweep(cfg, blk, n, dms, on_device=True)
        plain.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        ctx.process_block_dm_sweep(cfg, blk, n, dms, on_device=True, outputs=True, h_series=h_series,
                                   d_spectrum=d_spec)
        ex.append(time.perf_counter() - t0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    p_ms, e_ms = 1e3 * float(np.median(plain)), 1e3 * float(np.median(ex))
    print(json.dumps({"workload": f"config4 shape: 2^{log2n} samples x {len(dms)} trial DMs", "reps": reps,
                      "plain_ms_per_block": p_ms, "outputs_ms_per_block": e_ms, "outputs_over_plain": e_ms / p_ms,
                      "one_trial_share": 1.0 / len(dms), "plain_ms_all": [1e3 * t for t in plain],
                      "outputs_ms_all": [1e3 * t for t in ex], "card": card}))
    sys.exit(0)
t0 = time.perf_counter()
for _ in range(reps):
    res = ctx.process_block_dm_sweep(cfg, blk, n, dms, on_device=True)
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / reps
print(json.dumps({"workload": f"config4 shape: 2^{log2n} samples x {len(dms)} trial DMs", "ms_per_block": dt * 1e3,
                  "ms_per_trial": dt * 1e3 / len(dms), "trial_gsamples_per_s": n * len(dms) / dt / 1e9,
                  "block_gsamples_per_s": n / dt / 1e9}))
