#!/usr/bin/env python
"""Per-kernel times of BASELINE config #3 (two polarisations of 2^26 8-bit samples, rows of 2^14: the sweep-order
route, DESIGN §5). Every launch of a block's per-stream chain is timed alone: SRTB_B200_LANES=1 keeps both streams on
one CUDA stream, so no two big kernels overlap. Input is bench.py's ring of distinct seeded blocks (larger than L2),
submitted device-resident through the ring API as bench.py does; kernel times come from torch.profiler (CUDA
activities) in a run of its own after a warm-up.

For each kernel: launches per stream per block, µs per launch, the bytes it must move per launch (HBM, from the
shapes), GB/s and the share of the 3.35 TB/s data-sheet bandwidth. A control row times the row sweep's body without
the split or the cluster: the forward C2C of the same [P][L] rows in place (values are not looked at). The card's name
and power limit are read in the same run.  usage: config3_kernels.py [--steps K] [--warmup W] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

os.environ["SRTB_B200_LANES"] = "1"   # read when a context is created

import torch  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
import bench  # noqa: E402
import srtb_b200  # noqa: E402

DATASHEET_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[torch.cuda.current_device()].split(",")]
        return name, power
    except Exception:  # noqa: BLE001 - the table is still worth printing without the power limit
        return torch.cuda.get_device_name(), "unknown"


def bytes_per_launch(name, n):
    """HBM bytes a launch must move for one stream of n samples (M = n / 2 complex bins, 8 bytes each)"""
    if name.startswith("r2c_raw_col2048_kernel"):
        return 2 * n + 4 * n          # both polarisations' 8-bit samples in (the 32-byte raw rows), the [P][L] scratch out
    if name.startswith("r2c_rows_split_kernel"):
        return 4 * n + 4 * n          # scratch in, spectrum out
    if name.startswith("waterfall_sweep_order_kernel"):
        return 4 * n + 4 * n          # spectrum in, dynamic spectrum out (the chirp phase is computed, not read)
    return None                       # zap ranges and the detector tail: no streaming traffic of their own


def kernel_times(prof):
    """kernel name -> [launches, total µs] of the CUDA activities of a profile"""
    acc = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or not e.device_time:
            continue
        name = e.name.split("(")[0].split("<")[0].replace("void ", "").replace("srtb_b200::", "").strip()
        acc[name][0] += 1
        acc[name][1] += e.device_time
    return acc


def control_c2c(n, steps, warmup):
    """µs per launch of the row sweep's body without the split or the cluster: the forward C2C of the same [P][L]
    rows (fft_bigrow_kernel<14, true, false, 0>, in place, 8 + 8 bytes per point), timed the same way"""
    L = 1 << 14
    P = n // 2 // L
    x = torch.randn(P * L * 2, device="cuda", dtype=torch.float32)   # 16-byte aligned: the one-sweep route
    ctx = srtb_b200.Context(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    try:
        for _ in range(warmup):
            ctx.fft_c2c(x, L, P, +1)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                ctx.fft_c2c(x, L, P, +1)
            torch.cuda.synchronize()
    finally:
        ctx.close()
    cnt, us = kernel_times(prof)["fft_bigrow_kernel"]
    return us / cnt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    w = bench.WORKLOADS["config3"]
    H = bench.Harness(torch, srtb_b200, "config3", w, n_contexts=1, rank=0, local_rank=0, inject_pulse=True)
    n, streams = H.n, H.streams
    H.warm(H.step_device, args.warmup)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            H.step_device(i)
        H.drain()
        torch.cuda.synchronize()
    H.close()
    acc = kernel_times(prof)
    total_us = sum(cnt * (us / cnt) for cnt, us in acc.values()) / args.steps
    ctl = control_c2c(n, args.steps, args.warmup)
    name, power = card()
    launches = args.steps * streams
    rows = []
    for k, (cnt, us) in sorted(acc.items(), key=lambda kv: -kv[1][1]):
        per = us / cnt
        b = bytes_per_launch(k, n)
        row = {"kernel": k, "per_stream_block": cnt / launches, "us": per}
        if b:
            row.update(bytes=b, gbs=b / (per * 1e-6) / 1e9, share=b / (per * 1e-6) / DATASHEET_BPS)
        rows.append(row)
    b = bytes_per_launch("r2c_rows_split_kernel", n)
    rows.append({"kernel": "control: same body, C2C, no split", "per_stream_block": 1.0, "us": ctl, "bytes": b,
                 "gbs": b / (ctl * 1e-6) / 1e9, "share": b / (ctl * 1e-6) / DATASHEET_BPS})
    print(f"config #3, {streams} streams of 2^{n.bit_length() - 1} samples, one lane; {args.steps} blocks profiled")
    print(f"card: {name}, power limit {power}")
    print(f"{'kernel':34s} {'/stream':>7s} {'us':>9s} {'MB':>8s} {'GB/s':>8s} {'of 3.35 TB/s':>12s}")
    for r in rows:
        mb = f"{r['bytes'] / 1e6:8.1f}" if "bytes" in r else f"{'-':>8s}"
        gbs = f"{r['gbs']:8.0f}" if "bytes" in r else f"{'-':>8s}"
        sh = f"{r['share']:12.3f}" if "bytes" in r else f"{'-':>12s}"
        print(f"{r['kernel'][:34]:34s} {r['per_stream_block']:7.2f} {r['us']:9.1f} {mb} {gbs} {sh}")
    print(f"device time per block (both streams, all activities): {total_us / 1e3:.3f} ms")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "kernels": rows,
                                               "device_ms_per_block": total_us / 1e3}, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
