#!/usr/bin/env python
"""Times srtb_b200_incoherent_dm_search at the config #3 stream shape (2^26 samples: C = 2^11 channels of L = 2^14)
for 64, 256 and 1024 trial DMs spread over dm +- 1 pc cm^-3, on a random dynamic spectrum already on the device.
CUDA events around each call (the call synchronises once), 3 warm-up calls, the median of --reps (default 10).
Per run: ms per call, adds/s (n_dm * C * T adds), spectrum bytes read by the dedispersion kernel, and the card with its
power limit read in the same run. Beside it, tools/dm_sweep_bench.py's coherent ms per trial at the same shape, and
whether 1024 incoherent trials take less time than 16 coherent ones. Prints one JSON line."""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
import srtb_b200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--trials", default="64,256,1024")
ap.add_argument("--no-coherent", action="store_true", help="skip the coherent per-trial reference")
args = ap.parse_args()

torch.cuda.set_device(0)
ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
log2n, C_ = 26, 1 << 11
L = (1 << (log2n - 1)) // C_
f_low, bw, sr, dm = 1000.0, 500.0, 1e9, 100.0
g = torch.Generator(device="cuda").manual_seed(0)
x = torch.randn((C_, L, 2), device="cuda", generator=g, dtype=torch.float32)
x[7].zero_()  # one flagged channel, as SK leaves them

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
runs = []
for n_dm in [int(v) for v in args.trials.split(",")]:
    dms = list(dm + np.linspace(-1.0, 1.0, n_dm))
    h_series = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
    for _ in range(3):
        res, _, _, _ = ctx.incoherent_dm_search(x, L, C_, 0, f_low, bw, sr, dm, dms, 8.0, 0.9, 256, h_series)
    T = res[0].time_series_count
    # the timed call is the C entry alone, with its buffers made beforehand (the Python wrapper's conversion of 1024
    # peak records to numpy costs milliseconds of host time)
    arr = (C.c_float * n_dm)(*dms)
    c_res = (srtb_b200.DetectResult * n_dm)()
    c_peaks = (srtb_b200.Peak * n_dm)()
    best = C.c_int32()
    times = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = ctx.lib.srtb_b200_incoherent_dm_search(ctx.h, x.data_ptr(), L, C_, 0, f_low, bw, sr, dm, arr, n_dm, 8.0,
                                                    0.9, 256, c_res, C.cast(c_peaks, C.c_void_p), C.byref(best),
                                                    h_series.ctypes.data)
        e1.record()
        assert rc == 0, rc
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    _, sp, sm = srtb_b200.incoherent_shifts(C_, f_low, bw, sr, dm, dms, table=False)
    adds = n_dm * C_ * T
    runs.append({"n_dm": n_dm, "T": T, "s_plus": sp, "s_minus": sm, "ms_per_call": ms, "ms_all": times,
                 "adds_per_s": adds / (ms * 1e-3),
                 # the spectrum once; each group of up to 64 trials re-reads the span of every channel it needs
                 "spectrum_bytes": C_ * L * 8, "spectrum_bytes_read_by_groups_max": -(-n_dm // 64) * C_ * L * 8})
out = {"workload": f"incoherent DM search, config #3 stream shape: 2^{log2n} samples, C = {C_}, L = {L}",
       "card": card, "runs": runs}
if not args.no_coherent:
    r = subprocess.run([sys.executable, str(ROOT / "tools" / "dm_sweep_bench.py"), str(log2n), "5"],
                       capture_output=True, text=True)
    if r.returncode == 0:
        coh = json.loads(r.stdout.strip().splitlines()[-1])
        out["coherent_ms_per_trial"] = coh["ms_per_trial"]
        big = [run for run in runs if run["n_dm"] == 1024]
        if big:
            out["target_1024_incoherent_below_16_coherent"] = big[0]["ms_per_call"] < 16 * coh["ms_per_trial"]
            out["ratio_1024_incoherent_to_16_coherent"] = big[0]["ms_per_call"] / (16 * coh["ms_per_trial"])
    else:
        out["coherent_error"] = r.stderr[-500:]
print(json.dumps(out))
ctx.close()
