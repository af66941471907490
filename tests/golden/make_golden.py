#!/usr/bin/env python
"""Generates tests/golden/srtb_golden.npz, srtb_chain_golden.npz and srtb_ref_vectors.npz from the REFERENCE'S OWN
code (oracle/_ref/libsrtb_ref.so, the reference headers compiled through oracle/ref_shim). Run where the reference
source tree is at hand:   make -C oracle ref REF=<reference>/userspace && python tests/golden/make_golden.py
The tests read only the committed .npz files."""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import ref_lib  # noqa: E402


def main():
    ref = ref_lib.load()
    assert ref is not None, "build oracle/_ref first: make -C oracle ref"
    rng = np.random.default_rng(20260921)
    g = {}
    raw = rng.integers(0, 256, 512, dtype=np.uint8)
    g["unpack_raw"] = raw
    for bits in (1, 2, 4, 8, -8, 16, -16):
        g[f"unpack_b{bits}"] = ref.unpack(raw, raw.size * 8 // abs(bits), bits)
    g["unpack_b-8_hamming"] = ref.unpack(raw, raw.size, -8, 2)
    g["unpack_b2_hann"] = ref.unpack(raw, raw.size * 4, 2, 1)
    a, b = ref.unpack_interleaved_2(raw, raw.size // 2, -8)
    g["il2_a"], g["il2_b"] = a, b
    a, b = ref.unpack_snap1(raw, raw.size // 2)
    g["snap1_a"], g["snap1_b"] = a, b
    for s in (2, 4):
        for i, o in enumerate(ref.unpack_gznupsr_a1(raw, raw.size // s, s)):
            g[f"gznu{s}_{i}"] = o
    for w in (1, 2):
        g[f"window{w}_16"] = np.array([ref.window(w, i, 16) for i in range(16)], np.float32)
    x = (rng.uniform(-1, 1, 256) + 1j * rng.uniform(-1, 1, 256)).astype(np.complex64)
    g["fft_x"] = x
    g["fft_fwd"] = ref.fft_c2c(x, 1)
    g["fft_bwd"] = ref.fft_c2c(x, -1)
    xr = rng.integers(-128, 128, 512).astype(np.float32)
    g["r2c_x"] = xr
    g["r2c_X"] = ref.fft_r2c(xr)
    g["watfft_8x32"] = ref.watfft(x, 32, 8)
    spec = ((rng.standard_normal(2048) + 1j * rng.standard_normal(2048)) * 100).astype(np.complex64)
    spec[rng.integers(0, 2048, 8)] *= 40
    g["s1_x"] = spec
    g["s1_y"] = ref.rfi_s1_pipe(spec, 1.5, 16, 1000.0, 500.0, "1100-1110, 1300.5-1302")
    y = (rng.standard_normal(2048) + 1j * rng.standard_normal(2048)).astype(np.complex64)
    g["dd_x"] = y
    for tag, (fl, bw, dm) in {"a": (1000.0, 500.0, 56.778), "b": (1000.0, 400.0, 562.05), "c": (1437.0, -64.0, -478.80)}.items():
        g[f"dd_{tag}"] = ref.dedisperse_pipe(y, fl, bw, dm)
        g[f"dd_{tag}_params"] = np.array([fl, bw, dm], np.float64)
    C_, L = 16, 256
    d = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    d[2, :] = 3
    d[5, ::8] *= 9
    d[7, :] = 0
    g["s2_x"] = d.reshape(-1)
    g["s2_y"] = ref.rfi_s2_pipe(d.reshape(-1), L, C_, 1.2)
    e = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    e[:, 40:48] *= 10
    e[3, :] = 0
    g["det_x"] = e.reshape(-1)
    hs = ref.signal_detect_pipe(e.reshape(-1), L, C_, 2 * C_ * L, False, 1000.0, 500.0, 1e9, 0.0, 6.0, 0.9, 32)
    g["det_boxcar"] = np.array([h["boxcar"] for h in hs], np.int64)
    g["det_count"] = np.array([h["count"] for h in hs], np.int64)
    g["det_length"] = np.array([h["length"] for h in hs], np.int64)
    for h in hs:
        g[f"det_series_{h['boxcar']}"] = h["series"]
    np.savez_compressed(HERE / "srtb_golden.npz", **g)
    print("wrote", HERE / "srtb_golden.npz", sum(v.nbytes for v in g.values()), "bytes in", len(g), "arrays")
    chain_golden(ref)


def chain_golden(ref):
    """One block through the reference's pipes composed as main.cpp:170-204 wires them (every stage = the reference's
    own code through the shim): the fixture the GPU box checks srtb_b200_process_block against."""
    rng = np.random.default_rng(20260922)
    n, C_, dm = 1 << 15, 16, 0.0
    nc, L = n // 2, n // 2 // C_
    v = np.clip(np.round(rng.standard_normal(n) * 20), -127, 127)
    v[n // 2:n // 2 + 48] += np.round(rng.standard_normal(48) * 90)
    raw = np.clip(v, -127, 127).astype(np.int8).view(np.uint8)
    f_low, bw, fs, avg_thr, sk_thr, snr, chan_thr, maxbox = 1000.0, 500.0, 1e9, 5.0, 1.3, 6.0, 0.9, 64
    spec = ref.fft_r2c(ref.unpack(raw, n, -8))[:nc]
    spec = ref.rfi_s1_pipe(spec, avg_thr, C_, f_low, bw, "1200-1201")
    spec = ref.dedisperse_pipe(spec, f_low, bw, dm)
    spec = ref.watfft(spec, L, C_)
    spec = ref.rfi_s2_pipe(spec, L, C_, sk_thr)
    hs = ref.signal_detect_pipe(spec, L, C_, n, False, f_low, bw, fs, dm, snr, chan_thr, maxbox)
    g = {"raw": raw, "params": np.array([n, C_, dm, f_low, bw, fs, avg_thr, sk_thr, snr, chan_thr, maxbox], np.float64),
         "freq_pairs": np.array([1200.0, 1201.0], np.float32), "spectrum": spec.reshape(C_, L),
         "zero_count": np.array([int(np.sum(np.abs(spec.reshape(C_, L)[:, 0]) ** 2 == 0))], np.int64),
         "det_boxcar": np.array([h["boxcar"] for h in hs], np.int64),
         "det_count": np.array([h["count"] for h in hs], np.int64),
         "det_length": np.array([h["length"] for h in hs], np.int64)}
    np.savez_compressed(HERE / "srtb_chain_golden.npz", **g)
    print("wrote", HERE / "srtb_chain_golden.npz", sum(v_.nbytes for v_ in g.values()), "bytes;",
          "candidates at boxcars", g["det_boxcar"].tolist(), "counts", g["det_count"].tolist())
    ref_vectors(ref)


def _store_holders(g, key, hs, series_for=None):
    g[f"{key}_boxcar"] = np.array([h["boxcar"] for h in hs], np.int64)
    g[f"{key}_length"] = np.array([h["length"] for h in hs], np.int64)
    g[f"{key}_count"] = np.array([h["count"] for h in hs], np.int64)
    for h in hs:
        if series_for is None or h["boxcar"] in series_for:
            g[f"{key}_series_{h['boxcar']}"] = h["series"]


def ref_vectors(ref):
    """the reference's outputs for the seeded inputs of tests/test_oracle_vs_ref.py"""
    import test_oracle_vs_ref as t
    g = {}
    for bits in t.UNPACK_BITS:
        raw, n = t.unpack_input(bits)
        g[f"unpack_{bits}"] = t.digest(ref.unpack(raw, n, bits))
        if bits in (1, 2, 4):
            g[f"unpack_handwritten_{bits}"] = t.digest(ref.unpack_handwritten(raw, n, bits))
    raw = t.multistream_input()
    for bits in (8, -8, 16, -16):
        g[f"il2_{bits}"] = t.digests(ref.unpack_interleaved_2(raw, raw.size * 8 // abs(bits) // 2, bits))
    g["snap1"] = t.digests(ref.unpack_snap1(raw, raw.size // 2))
    for s in (2, 4):
        g[f"gznupsr_a1_{s}"] = t.digests(ref.unpack_gznupsr_a1(raw, raw.size // s, s))
    for w in (0, 1, 2):
        for n in (16, 1000):
            g[f"window_{w}_{n}"] = np.array([ref.window(w, i, n) for i in range(n)], np.float32)
        g[f"window_unpack_{w}"] = t.digest(ref.unpack(t.window_unpack_input(), 512, -8, w))
    for k in t.FFT_K:
        x, xr, (length, batch) = t.fft_inputs(k)
        for d in (1, -1):
            g[f"fft_{k}_{d}"] = t.digest(ref.fft_c2c(x, d))
        g[f"r2c_{k}"] = t.digest(ref.fft_r2c(xr))
        g[f"watfft_{k}"] = t.digest(ref.watfft(x, length, batch))
    for nc, C_ in t.S1_CASES:
        r = ref.rfi_s1_pipe(t.s1_input(nc), 1.5, C_, 1000.0, 500.0, t.S1_RANGES)
        g[f"s1_{nc}_zero"] = np.packbits(r == 0)
        g[f"s1_{nc}_blocks"] = t.digests(r[b:b + t.S1_BLOCK] for b in range(0, nc, t.S1_BLOCK))
    for i, s in enumerate(t.RANGE_STRINGS):
        g[f"ranges_{i}"] = np.array(ref.eval_rfi_ranges(s), np.float32).reshape(-1, 2)
    g["manual_kat"] = t.digest(ref.rfi_manual(np.ones(1500, np.complex64), 0.0, 1499.0,
                                              ref.eval_rfi_ranges(t.RANGE_STRINGS[0])))
    for i, (pairs, fl, bw) in enumerate(t.MANUAL_CASES):
        g[f"manual_{i}"] = t.digest(ref.rfi_manual(np.ones(1 << 12, np.complex64), fl, bw, pairs))
    for i, (nc, f_low, bw, dm) in enumerate(t.DD_CASES):
        x = t.dd_input(nc)
        g[f"dd_pipe_{i}"] = t.digest(ref.dedisperse_pipe(x, f_low, bw, dm))
        g[f"dd_op_{i}"] = t.digest(ref.dedisperse(x, *t.dd_f32_params(f_low, bw, nc), dm))
    g["nsamps_reserved"] = np.array([ref.nsamps_reserved(*a) for a in t.NSAMPS_CASES], np.int64)
    C_, L = t.S2_SHAPE
    r = ref.rfi_s2_pipe(t.s2_input().reshape(-1), L, C_, t.S2_THR).reshape(C_, L)
    g["s2_zero_rows"], g["s2_rows"] = np.all(r == 0, axis=1), t.digests(r)
    f_low, bw, fs, dm, snr, chan_thr = t.SD_PARAMS
    for i, (C_, L, maxbox, reserve) in enumerate(t.SD_CASES):
        x = t.sd_input(C_, L).reshape(-1)
        _store_holders(g, f"sd_{i}", ref.signal_detect_pipe(x, L, C_, 2 * C_ * L, reserve, f_low, bw, fs, dm, snr,
                                                            chan_thr, maxbox))
    f_low, bw, fs, avg_thr, sk_thr, snr, chan_thr, maxbox = t.CHAIN_PARAMS
    for i, (logn, C_, dm, bits) in enumerate(t.CHAIN_CASES):
        n = 1 << logn
        nc, L = n // 2, n // 2 // C_
        spec = ref.fft_r2c(ref.unpack(t.chain_input(logn, C_, bits), n, bits))[:nc]   # fft_pipe.hpp:75-77: count = N/2
        spec = ref.rfi_s1_pipe(spec, avg_thr, C_, f_low, bw, t.CHAIN_RANGES)
        spec = ref.dedisperse_pipe(spec, f_low, bw, dm)
        spec = ref.watfft(spec, L, C_)
        spec = ref.rfi_s2_pipe(spec, L, C_, sk_thr)
        g[f"chain_{i}_spectrum"] = spec.reshape(C_, L)
        _store_holders(g, f"chain_{i}", ref.signal_detect_pipe(spec, L, C_, n, False, f_low, bw, fs, dm, snr, chan_thr,
                                                               maxbox), series_for=())
    for i, (nt, nf) in enumerate(t.SKV1_CASES):
        x = t.refft_layout_block(np.random.default_rng(nt + nf), nt, nf)
        r = ref.sk_v1(x.reshape(-1), nf, nt, t.SKV1_THR).reshape(nt, nf)
        g[f"skv1_{i}_zero_cols"], g[f"skv1_{i}_cols"] = np.all(r == 0, axis=0), t.digests(r.T)
    sk_thr, snr, chan_thr = t.SDV1_PARAMS
    for i, (nt, nf, maxbox) in enumerate(t.SDV1_CASES):
        x = t.refft_layout_block(np.random.default_rng(7 * nt + nf), nt, nf)
        rspec, hs = ref.signal_detect_pipe_v1(x.reshape(-1), nf, nt, sk_thr, snr, chan_thr, maxbox)
        g[f"sdv1_{i}_spectrum"] = t.digest(rspec)
        _store_holders(g, f"sdv1_{i}", hs, series_for=(1,))
    np.savez_compressed(HERE / "srtb_ref_vectors.npz", **g)
    print("wrote", HERE / "srtb_ref_vectors.npz", (HERE / "srtb_ref_vectors.npz").stat().st_size, "bytes in", len(g),
          "arrays")


if __name__ == "__main__":
    main()
