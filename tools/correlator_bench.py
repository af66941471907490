"""Times srtb_b200_correlate (the baseband correlator on device bytes) with CUDA events after warm-up, and prints one
JSON line for the card, then one per input size:

    python tools/correlator_bench.py [--sizes 28,30] [--calls 10] [--warmup 3]

compulsory bytes = 2 input_size (both inputs read once) + 4 M (the M = input_size / 2 magnitudes written);
`GBps` = those bytes over the time per call, `of_3.35TBps` = that rate over the H100 SXM data-sheet HBM3 bandwidth.
`sweep_bytes` = what the launched kernels read and write with the unpack fused into the R2C's first sweep: per input,
the first sweep reads input_size bytes and writes 8 M, every further R2C sweep reads and writes 8 M; the cross
spectrum reads 16 M and writes 8 M, each backward C2C sweep reads and writes 8 M, the magnitude reads 8 M and writes 4 M.
An M-point transform takes 2 sweeps from 2^15 up to 2^20 points, 3 up to 2^26 and 4 above (the plans of
fft_r2c_with_power_mean and fft_c2c_impl; below 2^15 points they differ, and sweep_bytes is not exact there).

The integrating mode instead times srtb_b200_correlate_accumulate over chunks of 2^chunk samples per input:

    python tools/correlator_bench.py --segment_size 12,14,16,20 [--bits 8,2] [--chunk 28] [--calls 10] [--warmup 3]

`input_GBps` = both inputs' bytes (2 * 2^chunk * |bits| / 8) over the time per call. `sweep_bytes` per call, from the
shapes, per sample pair (one complex element of the packed rows; 2^chunk of them over both inputs): the pack reads
2 |bits| / 8 and writes 8 bytes, each sweep of the Ls-point C2C reads and writes 16 (1 sweep up to 2^14 points, 2 up
to 2^20, 3 up to 2^26), and the split reads 8."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))

HBM_PEAK = 3.35e12


def sweeps(m: int) -> int:
    q = m.bit_length() - 1
    return 1 if q <= 14 else 2 if q <= 20 else 3 if q <= 26 else 4


def sweep_bytes(input_size: int) -> int:
    m = input_size // 2
    p = sweeps(m)
    r2c = input_size + 8 * m + (p - 1) * 16 * m
    return 2 * r2c + 24 * m + p * 16 * m + 12 * m


def segment_sweep_bytes(chunk: int, ls: int, bits: int) -> int:
    pairs = chunk  # K Ls / 2 sample pairs per input, two inputs
    return pairs * 2 * abs(bits) // 8 + pairs * (8 + 16 * sweeps(ls) + 8)


def bench_segments(a, ctx, stream):
    import torch
    chunk = 1 << a.chunk
    for bits in (int(b) for b in a.bits.split(",")):
        nbytes = chunk * abs(bits) // 8
        g = torch.Generator(device="cuda").manual_seed(bits)
        d_1 = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
        d_2 = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
        for q in (int(s) for s in a.segment_size.split(",")):
            ls = 1 << q
            k = chunk // ls
            acc = torch.zeros(ls // 2, dtype=torch.complex128, device="cuda")
            launches = ctx.launch_count
            ctx.correlate_accumulate(d_1, d_2, bits, ls, k, acc, reset=True)
            per_call = ctx.launch_count - launches
            for _ in range(a.warmup):
                ctx.correlate_accumulate(d_1, d_2, bits, ls, k, acc)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.calls):
                ctx.correlate_accumulate(d_1, d_2, bits, ls, k, acc)
            e1.record(stream)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / a.calls
            sweep = segment_sweep_bytes(chunk, ls, bits)
            print(json.dumps({"segment_size": f"2^{q}", "bits": bits, "samples_per_input": f"2^{a.chunk}",
                              "segments": k, "ms_per_call": round(ms, 3),
                              "input_GBps": round(2 * nbytes / ms / 1e6, 1), "sweep_bytes": sweep,
                              "sweep_GBps": round(sweep / ms / 1e6, 1),
                              "sweep_of_3.35TBps": round(sweep / ms / 1e-3 / HBM_PEAK, 3),
                              "kernels_per_call": per_call, "calls": a.calls}), flush=True)
            del acc
        del d_1, d_2


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="28,30", help="log2 of input_size, comma separated")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--segment_size", default=None,
                    help="log2 of the segment sizes, comma separated: time the integrating mode's accumulate instead")
    ap.add_argument("--bits", default="8,2", help="sample widths of the integrating mode")
    ap.add_argument("--chunk", type=int, default=28, help="log2 of the samples per input per accumulate call")
    a = ap.parse_args()
    import torch

    import srtb_b200
    assert torch.cuda.is_available(), "correlator_bench needs a CUDA device"
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    ctx = srtb_b200.Context(0, stream.cuda_stream)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": gpu_info()}), flush=True)
    if a.segment_size:
        bench_segments(a, ctx, stream)
        ctx.close()
        return
    for k in (int(s) for s in a.sizes.split(",")):
        n = 1 << k
        g = torch.Generator(device="cuda").manual_seed(k)
        d_1 = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
        d_2 = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
        out = torch.empty(n // 2, dtype=torch.float32, device="cuda")
        launches = ctx.launch_count
        ctx.correlate(d_1, d_2, n, out)
        per_call = ctx.launch_count - launches
        for _ in range(a.warmup):
            ctx.correlate(d_1, d_2, n, out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.calls):
            ctx.correlate(d_1, d_2, n, out)
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / a.calls
        compulsory = 2.0 * n + 4.0 * (n // 2)
        sweep = sweep_bytes(n)
        print(json.dumps({"input_size": f"2^{k}", "ms_per_call": round(ms, 3), "compulsory_bytes": compulsory,
                          "GBps": round(compulsory / ms / 1e6, 1),
                          "of_3.35TBps": round(compulsory / ms / 1e-3 / HBM_PEAK, 4),
                          "sweep_bytes": sweep, "sweep_GBps": round(sweep / ms / 1e6, 1),
                          "sweep_of_3.35TBps": round(sweep / ms / 1e-3 / HBM_PEAK, 3),
                          "kernels_per_call": per_call, "calls": a.calls}), flush=True)
        del d_1, d_2, out
    ctx.close()


if __name__ == "__main__":
    main()
