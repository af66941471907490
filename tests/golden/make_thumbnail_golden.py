"""Writes srtb_thumbnail_ref_vectors.npz: the reference's own waterfall thumbnail (resample_spectrum_3 with norm(),
simplify_spectrum_normalize_with_average_value, generate_pixmap) on the seeded geometries of
tests/thumbnail_oracle.py, run through the host SYCL shim (thumbnail_ref_driver.cpp).

    python tests/golden/make_thumbnail_golden.py --reference <reference checkout>/userspace

Only the outputs are stored; the inputs are regenerated from their seeds (an input checksum is stored with them)."""
from __future__ import annotations

import argparse
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(HERE.parent))
import thumbnail_oracle as T  # noqa: E402


def build(ref: Path, out: Path) -> C.CDLL:
    subprocess.run(["g++", "-O2", "-std=c++20", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-w", "-shared",
                    "-DSRTB_ENABLE_GUI=0", "-I", str(ROOT / "oracle" / "ref_shim"), "-I", str(ref / "include"),
                    "-I", str(ref / "3rdparty" / "dsmath"), "-I", str(ref / "3rdparty" / "concurrentqueue"),
                    "-o", str(out), str(HERE / "thumbnail_ref_driver.cpp")], check=True)
    lib = C.CDLL(str(out))
    P, SZ = C.c_void_p, C.c_size_t
    lib.srtb_ref_simplify_spectrum.argtypes = [P, SZ, SZ, SZ, SZ, P, P, P, P]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="the reference's userspace directory")
    ap.add_argument("--out", type=Path, default=HERE / "srtb_thumbnail_ref_vectors.npz")
    a = ap.parse_args()
    data = {}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build(a.reference, Path(tmp) / "libthumb_ref.so")
        for name, (Ch, L, H, W, _) in T.CASES.items():
            spec = T.case_spectrum(name)
            raw = np.zeros((H, W), np.float32)
            inten = np.zeros((H, W), np.float32)
            pix = np.zeros((H, W), np.uint32)
            avg = np.zeros(1, np.float32)
            assert lib.srtb_ref_simplify_spectrum(spec.ctypes.data, L, Ch, W, H, raw.ctypes.data, inten.ctypes.data,
                                                  pix.ctypes.data, avg.ctypes.data) == 0
            data[f"{name}__raw"] = raw
            data[f"{name}__intensity"] = inten
            data[f"{name}__pixmap"] = pix
            data[f"{name}__average"] = avg
            data[f"{name}__input_sum"] = np.array([np.sum(T.norm(spec), dtype=np.float64)])
            print(f"{name}: {Ch}x{L} -> {H}x{W}, average {avg[0]:.6g}")
    np.savez_compressed(a.out, **data)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
