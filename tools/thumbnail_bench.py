"""Times srtb_b200_simplify_spectrum (the waterfall thumbnail: three kernels) with CUDA events at the shapes the
project's configurations produce, and prints one JSON line per shape plus the card it ran on:

    python tools/thumbnail_bench.py [--calls 200] [--warmup 20]

compulsory bytes = 8 C L (the complex64 spectrum, read once) + 8 W H (intensity and pixmap written); GB/s = those bytes
over the time per call; `of_3.35TBps` = that rate over the H100 SXM data-sheet HBM3 bandwidth.

--executable-seconds S (S > 0) also runs the product executable (src/srtb_b200) on an unpaced synthetic stream of
2^26-sample blocks with 2048 channels (the config #5 source, as fast as the path takes it) for S seconds, with
gui_enable = 0 and = 1 alternately (two runs each, 1920 x 1080 pixmap), and prints the executable's sustained rate
and, with the thumbnail, how many thumbnails it wrote and how many blocks it skipped."""
from __future__ import annotations

import argparse
import json
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))

SHAPES = {  # name: (C, L, H, W)
    "config3 (2048 x 16384 -> 1080 x 1920)": (2048, 16384, 1080, 1920),
    "config1 (2048 x 2^18 -> 1080 x 1920)": (2048, 1 << 18, 1080, 1920),
}
HBM_PEAK = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def executable_run(gui: int, seconds: float, out_dir: Path) -> dict:
    exe = ROOT / "src" / "srtb_b200"
    cmd = [str(exe), "--config_file_name", str(out_dir / "none.cfg"), "--gpu_devices", "0", "--chains_per_gpu", "2",
           "--ring_depth", "3", "--discard_output", "1", "--synthetic_udp_rate", "0", "--synthetic_duration",
           repr(float(seconds)), "--baseband_input_count", "2 ** 26", "--baseband_input_bits", "-8",
           "--baseband_format_type", "fastmb_roach2", "--baseband_freq_low", "1000.0", "--baseband_bandwidth", "500.0",
           "--baseband_sample_rate", "1e9", "--dm", "56.778", "--baseband_reserve_sample", "0",
           "--spectrum_channel_count", "2048", "--mitigate_rfi_average_method_threshold", "5",
           "--mitigate_rfi_spectral_kurtosis_threshold", "1.05", "--signal_detect_signal_noise_threshold", "8",
           "--signal_detect_max_boxcar_length", "256", "--baseband_output_file_prefix", str(out_dir / "run_"),
           "--gui_enable", str(gui), "--gui_pixmap_width", "1920", "--gui_pixmap_height", "1080", "--log_level", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        raise SystemExit(f"srtb_b200 failed: {r.stderr[-1500:]}")
    res = json.loads([line for line in r.stdout.splitlines() if line.startswith("{")][-1])
    m = re.search(r"waterfall: (\d+) thumbnail\(s\) written, (\d+) block\(s\) skipped", r.stderr)
    out = {"gui_enable": gui, "gsamples_per_s": round(res["gsamples_per_s"], 3), "blocks": res["blocks"],
           "seconds": round(res["seconds"], 3)}
    if m:
        out.update(thumbnails_written=int(m.group(1)), blocks_skipped=int(m.group(2)),
                   ppm_files=sorted(p.name for p in out_dir.glob("*.ppm")))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--executable-seconds", type=float, default=0.0)
    a = ap.parse_args()
    import torch

    import srtb_b200
    assert torch.cuda.is_available(), "thumbnail_bench needs a CUDA device"
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    ctx = srtb_b200.Context(0, stream.cuda_stream)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": gpu_info()}), flush=True)
    for name, (C, L, H, W) in SHAPES.items():
        spec = torch.randn(C, L, dtype=torch.complex64, device="cuda")
        inten = torch.empty(H, W, dtype=torch.float32, device="cuda")
        pix = torch.empty(H, W, dtype=torch.int32, device="cuda")
        for _ in range(a.warmup):
            ctx.simplify_spectrum(spec, L, C, W, H, inten, pix)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.calls):
            ctx.simplify_spectrum(spec, L, C, W, H, inten, pix)
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / a.calls
        nbytes = 8.0 * C * L + 8.0 * W * H
        print(json.dumps({"shape": name, "ms_per_call": round(ms, 4), "compulsory_bytes": nbytes,
                          "GBps": round(nbytes / ms / 1e6, 1), "of_3.35TBps": round(nbytes / ms / 1e-3 / HBM_PEAK, 3),
                          "calls": a.calls}), flush=True)
        del spec, inten, pix
    ctx.close()
    if a.executable_seconds > 0:
        torch.cuda.empty_cache()
        for gui in (0, 1, 0, 1):
            with tempfile.TemporaryDirectory() as tmp:
                print(json.dumps({"executable": executable_run(gui, a.executable_seconds, Path(tmp))}), flush=True)


if __name__ == "__main__":
    main()
