"""Writes srtb_correlator_ref_vectors.npz: the output of the reference's own baseband correlator
(userspace/src/correlator.cpp, compiled unmodified through the host SYCL shim by correlator_ref_driver.cpp) on the
seeded input pairs of tests/correlator_oracle.py. Each pair is written as pol_1.bin / pol_2.bin into a temporary
working directory, where the program reads them.

    python tests/golden/make_correlator_golden.py --reference <reference checkout>/userspace

Only the outputs are stored; the inputs are regenerated from their seeds (their CRC-32s are stored with them)."""
from __future__ import annotations

import argparse
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(HERE.parent))
import correlator_oracle as K  # noqa: E402


def build(ref: Path, out: Path) -> Path:
    subprocess.run(["g++", "-O2", "-std=c++20", "-ffp-contract=off", "-fno-fast-math", "-w", "-DSRTB_ENABLE_GUI=0",
                    "-I", str(HERE / "correlator_shim"), "-I", str(ROOT / "oracle" / "ref_shim"),
                    "-I", str(ref / "include"), "-I", str(ref / "3rdparty" / "dsmath"),
                    "-I", str(ref / "3rdparty" / "concurrentqueue"), "-I", str(ref / "src"),
                    "-o", str(out), str(HERE / "correlator_ref_driver.cpp")], check=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="the reference's userspace directory")
    ap.add_argument("--out", type=Path, default=HERE / "srtb_correlator_ref_vectors.npz")
    a = ap.parse_args()
    data = {}
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        exe = build(a.reference, tmp / "correlator_ref")
        for name in K.CASES:
            in_1, in_2 = K.case_inputs(name)
            work = tmp / name
            work.mkdir()
            in_1.tofile(work / "pol_1.bin")
            in_2.tofile(work / "pol_2.bin")
            subprocess.run([str(exe), str(work / "corr.bin")], cwd=work, check=True, capture_output=True)
            out = np.fromfile(work / "corr.bin", np.float32)
            assert out.size == K.sizes(min(in_1.size, in_2.size))[0], (name, out.size)
            data[f"{name}__out"] = out
            data[f"{name}__input_crc"] = np.array([K.checksum(in_1), K.checksum(in_2)], np.uint64)
            print(f"{name}: {in_1.size} and {in_2.size} bytes -> {out.size} floats")
    np.savez_compressed(a.out, **data)
    print(f"wrote {a.out} ({a.out.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
