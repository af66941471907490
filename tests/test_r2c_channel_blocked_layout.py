"""The channel-blocked spectrum of the config-#3 route on the CPU: its index algebra against numpy.fft.rfft
(tools/proto_r2c_sweep_order.py), and no local memory (register spills) in the three kernels of the route, read with
cuobjdump -res-usage from the built library."""
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import proto_r2c_sweep_order as proto  # noqa: E402

LIB = ROOT / "simple-radio-telescope-backend_b200" / "csrc" / "libsrtb_b200.so"
KERNELS = ("r2c_raw_col2048_kernel", "r2c_rows_split_kernel", "waterfall_sweep_order_kernel")


def test_channel_blocked_index_algebra():
    assert proto.main_channel_blocked(5, 8) == 0


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump not installed")
    return tool


def test_sweep_order_kernels_use_no_local_memory():
    assert LIB.exists(), "build() leaves the library in csrc/"
    out = subprocess.run([_cuobjdump(), "-res-usage", str(LIB)], capture_output=True, text=True, check=True).stdout
    seen = {k: 0 for k in KERNELS}
    lines = out.splitlines()
    for i, ln in enumerate(lines):
        m = re.search(r"Function (\S+):", ln)
        if not m:
            continue
        hit = [k for k in KERNELS if k in m.group(1)]
        if not hit:
            continue
        usage = ln + " " + (lines[i + 1] if i + 1 < len(lines) else "")
        local = re.search(r"LOCAL:(\d+)", usage)
        stack = re.search(r"STACK:(\d+)", usage)
        assert local and stack, usage
        assert int(local.group(1)) == 0 and int(stack.group(1)) == 0, (hit[0], usage)
        seen[hit[0]] += 1
    assert all(seen.values()), seen
