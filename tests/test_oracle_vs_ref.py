"""Pins the CPU oracle (oracle/srtb_oracle.cpp) against the reference's own operator/pipe headers, compiled through
the host shim (oracle/_ref/libsrtb_ref.so, see oracle/ref_shim/README.md). The reference's outputs for the seeded
inputs below are stored in tests/golden/srtb_ref_vectors.npz (tests/golden/make_golden.py writes them), so the
comparison needs neither the reference tree nor the shim library. Bit-exact wherever the reference's arithmetic
order is fully specified (stored as SHA-256 digests of the reference's bytes, per row or block where only some rows
are compared), tolerance only where a reduction's order is the runtime's choice."""
import hashlib
from pathlib import Path

import numpy as np
import pytest

VEC_PATH = Path(__file__).resolve().parent / "golden" / "srtb_ref_vectors.npz"
S1_BLOCK = 1024   # elements per digest of the s1 pipe's output


def digest(a) -> str:
    """SHA-256 (first 128 bits) of an array's bytes; -0.0 counts as 0.0 (a zapped element is zero either way)"""
    a = np.ascontiguousarray(a)
    if a.dtype.kind in "fc":
        a = a + np.zeros(1, a.dtype)
    return hashlib.sha256(a.tobytes()).hexdigest()[:32]


def digests(rows) -> np.ndarray:
    return np.array([digest(r) for r in rows])


def rel(a, b):
    a, b = np.asarray(a).astype(np.complex128).ravel(), np.asarray(b).astype(np.complex128).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(scope="module")
def V():
    return np.load(VEC_PATH)


def holders(V, key):
    """the reference's detector output (signal_detect_pipe holders) as stored"""
    out = []
    for bc, ln, cnt in zip(V[f"{key}_boxcar"], V[f"{key}_length"], V[f"{key}_count"]):
        s = f"{key}_series_{int(bc)}"
        out.append(dict(boxcar=int(bc), length=int(ln), count=int(cnt), series=V[s] if s in V.files else None))
    return out


# ---- seeded inputs (tests/golden/make_golden.py runs the reference on exactly these)
UNPACK_BITS = [1, 2, 4, 8, -8, 16, -16, 32, 64]
FFT_K = [1, 4, 10, 14]
S1_CASES = [(1 << 10, 16), ((1 << 14) + 3, 64), (1 << 18, 2048)]
S1_RANGES = "1100-1101, 1300.5-1302"
RANGE_STRINGS = ["11-12, 15-90, 233-235, 1176-1177", "", "1418-1422", "1-2-3, 5-6", " 7 - 8 ,9-10", "3-4,"]
MANUAL_CASES = [([(1418.0, 1422.0)], 1437.0, -64.0), ([(1422.0, 1418.0)], 1437.0, -64.0),
                ([(100.0, 200.0)], 1000.0, 500.0), ([(1400.0, 1600.0)], 1000.0, 500.0)]
DD_CASES = [(1 << 14, 1000.0, 500.0, 56.778), ((1 << 12) + 1, 1000.0, 400.0, 562.05),
            (1 << 16, 1437.0, -64.0, -478.80), (1 << 10, 1000.0, 500.0, 0.0)]
NSAMPS_CASES = [(1 << 26, 1 << 11, 1000.0, 500.0, 1e9, 5.0, True), (1 << 24, 1 << 11, 1000.0, 500.0, 1e9, 56.778, True),
                (1 << 30, 1 << 11, 1437.0, -64.0, 128e6, -478.80, True),
                (1 << 30, 1 << 11, 1437.0, -64.0, 128e6, -478.80, False),
                (1 << 28, 1 << 15, 1000.0, 500.0, 1e9, 100.0, True), (1 << 28, 1 << 15, 1000.0, 500.0, 1e9, 1.0, True)]
S2_SHAPE, S2_THR = (48, 1024), 1.05
SD_CASES = [(16, 256, 16, False), (64, 2048, 256, False), (32, 1000, 64, True)]
SD_PARAMS = (1000.0, 500.0, 1e9, 0.005, 6.0, 0.9)            # f_low, bw, fs, dm, snr, chan_thr
CHAIN_CASES = [(14, 16, 0.0, -8), (15, 32, 0.02, -8), (14, 8, 0.0, 2)]
CHAIN_PARAMS = (1000.0, 500.0, 1e9, 5.0, 1.3, 6.0, 0.9, 32)  # f_low, bw, fs, avg_thr, sk_thr, snr, chan_thr, maxbox
CHAIN_RANGES = "1200-1201"
SKV1_CASES, SKV1_THR = [(256, 64), (1000, 48)], 1.1
SDV1_CASES, SDV1_PARAMS = [(512, 64, 32), (1000, 128, 256)], (1.4, 5.0, 0.9)   # sk_thr, snr, chan_thr


def unpack_input(bits):
    rng = np.random.default_rng(abs(bits))
    nbytes = 1 << 12
    raw = (rng.standard_normal(nbytes // 4).astype(np.float32).view(np.uint8) if bits == 32 else
           rng.standard_normal(nbytes // 8).view(np.uint8) if bits == 64 else rng.integers(0, 256, nbytes, dtype=np.uint8))
    return raw, nbytes * 8 // abs(bits)


def multistream_input():
    return np.random.default_rng(9).integers(0, 256, 1 << 13, dtype=np.uint8)


def window_unpack_input():
    return np.random.default_rng(3).integers(0, 256, 512, dtype=np.uint8)


def fft_inputs(k):
    rng = np.random.default_rng(k)
    n = 1 << k
    x = (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)
    xr = rng.uniform(-1, 1, 2 * n).astype(np.float32)
    return x, xr, (n // 2 if n > 1 else 1, 2 if n > 1 else 1)


def s1_input(nc):
    rng = np.random.default_rng(nc)
    x = ((rng.standard_normal(nc) + 1j * rng.standard_normal(nc)) * 100).astype(np.complex64)
    x[rng.integers(0, nc, 12)] *= 40
    return x


def dd_input(nc):
    rng = np.random.default_rng(nc)
    return (rng.standard_normal(nc) + 1j * rng.standard_normal(nc)).astype(np.complex64)


def dd_f32_params(f_low, bw, nc):
    f_min, f_c = np.float32(f_low), np.float32(np.float32(f_low) + np.float32(bw))
    df = np.float32(np.float32(bw) / np.float32(nc))
    return float(f_min), float(f_c), float(df)


def s2_input():
    rng = np.random.default_rng(21)
    C_, L = S2_SHAPE
    x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    x[5, :] = 3
    x[9, ::8] *= 9
    x[11, :] = 0
    return x


def sd_input(C_, L):
    rng = np.random.default_rng(C_ * L)
    x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
    x[:, L // 8:L // 8 + 8] *= 10
    x[1, :] = 0
    return x


def chain_input(logn, C_, bits):
    n = 1 << logn
    rng = np.random.default_rng(logn * 7 + C_)
    if bits == -8:
        v = np.clip(np.round(rng.standard_normal(n) * 20), -127, 127)
        v[n // 2:n // 2 + 32] += np.round(rng.standard_normal(32) * 90)
        return np.clip(v, -127, 127).astype(np.int8).view(np.uint8)
    return rng.integers(0, 256, n * bits // 8, dtype=np.uint8)


def refft_layout_block(rng, nt, nf):
    """spectra [time][frequency]: noise, one steady tone (low kurtosis), one bursty channel (high kurtosis), one
    manually zapped channel, and a broadband burst over a few consecutive spectra"""
    x = (rng.standard_normal((nt, nf)) + 1j * rng.standard_normal((nt, nf))).astype(np.complex64)
    x[:, 5] = 3
    x[::8, 9] *= 9
    x[:, 11] = 0
    x[nt // 3:nt // 3 + 16, :] *= 1.6   # mild enough to stay inside the kurtosis thresholds of the detector tests
    return x


# ---- the comparisons
@pytest.mark.parametrize("bits", UNPACK_BITS)
def test_unpack_bit_exact(oracle, V, bits):
    raw, n = unpack_input(bits)
    o = oracle.unpack(raw, n, bits)
    assert digest(o) == V[f"unpack_{bits}"]
    if bits in (1, 2, 4):     # generic == handwritten, as test-unpack.cpp:211-254 checks
        assert digest(o) == V[f"unpack_handwritten_{bits}"]


def test_unpack_multistream_bit_exact(oracle, V):
    raw = multistream_input()
    for bits in (8, -8, 16, -16):
        n = raw.size * 8 // abs(bits) // 2
        assert [digest(a) for a in oracle.unpack_interleaved_2(raw, n, bits)] == list(V[f"il2_{bits}"])
    assert [digest(a) for a in oracle.unpack_snap1(raw, raw.size // 2)] == list(V["snap1"])
    for streams in (2, 4):
        outs = oracle.unpack_gznupsr_a1(raw, raw.size // streams, streams)
        assert [digest(a) for a in outs] == list(V[f"gznupsr_a1_{streams}"])


@pytest.mark.parametrize("window", [0, 1, 2])
def test_window_bit_exact(oracle, V, window):
    for n in (16, 1000):
        got = np.array([oracle.window(window, i, n) for i in range(n)], np.float32)
        assert np.array_equal(got, V[f"window_{window}_{n}"])
    raw = window_unpack_input()
    assert digest(oracle.unpack(raw, 512, -8, window)) == V[f"window_unpack_{window}"]


@pytest.mark.parametrize("k", FFT_K)
def test_naive_fft_bit_exact(oracle, V, k):
    x, xr, (length, batch) = fft_inputs(k)
    for d in (1, -1):
        assert digest(oracle.fft_c2c(x, d)) == V[f"fft_{k}_{d}"]
    assert digest(oracle.fft_r2c(xr)) == V[f"r2c_{k}"]
    assert digest(oracle.watfft(x, length, batch)) == V[f"watfft_{k}"]


@pytest.mark.parametrize("nc,C_", S1_CASES)
def test_rfi_s1_pipe(oracle, V, nc, C_):
    x = s1_input(nc)
    thr = 1.5
    rzero = np.unpackbits(V[f"s1_{nc}_zero"], count=nc).astype(bool)
    o, mean, mask = oracle.rfi_s1_average(x, thr, C_)
    o = oracle.rfi_manual(o, 1000.0, 500.0, oracle.eval_rfi_ranges(S1_RANGES))
    p = np.abs(x.astype(np.complex128)) ** 2
    border = np.abs(p / (thr * p.mean()) - 1) < 1e-4       # the mean's summation order is the runtime's
    assert np.array_equal(rzero[~border], (o == 0)[~border])
    # normalised values are bit-identical: every block whose zap decisions agree has the reference's bytes
    nb = (nc + S1_BLOCK - 1) // S1_BLOCK
    same = [np.array_equal(rzero[b * S1_BLOCK:(b + 1) * S1_BLOCK], (o == 0)[b * S1_BLOCK:(b + 1) * S1_BLOCK])
            for b in range(nb)]
    got =digests(o[b * S1_BLOCK:(b + 1) * S1_BLOCK] for b in range(nb))
    assert np.array_equal(got[same], V[f"s1_{nc}_blocks"][same])
    assert ((o == 0) & (x != 0)).sum() >= 10


def test_rfi_ranges_and_manual_zap(oracle, V):
    for i, s in enumerate(RANGE_STRINGS):
        assert oracle.eval_rfi_ranges(s) == [tuple(map(float, r)) for r in V[f"ranges_{i}"]], s
    x = np.ones(1500, np.complex64)
    rr = [tuple(map(float, r)) for r in V["ranges_0"]]
    assert digest(oracle.rfi_manual(x, 0.0, 1499.0, rr)) == V["manual_kat"]
    x = np.ones(1 << 12, np.complex64)
    for i, (pairs, fl, bw) in enumerate(MANUAL_CASES):
        assert digest(oracle.rfi_manual(x, fl, bw, pairs)) == V[f"manual_{i}"]


@pytest.mark.parametrize("nc,f_low,bw,dm", DD_CASES)
def test_dedisperse_pipe_bit_exact(oracle, V, nc, f_low, bw, dm):
    case = DD_CASES.index((nc, f_low, bw, dm))
    f_min, f_c, df = dd_f32_params(f_low, bw, nc)
    o = digest(oracle.dedisperse(dd_input(nc), f_min, f_c, df, dm))
    assert o == V[f"dd_pipe_{case}"]       # the reference's dedisperse pipe
    assert o == V[f"dd_op_{case}"]         # and its operator called with the pipe's float32 parameters


def test_nsamps_reserved(oracle, V):
    assert [oracle.nsamps_reserved(*args) for args in NSAMPS_CASES] == V["nsamps_reserved"].tolist()


def test_rfi_s2_pipe(oracle, V):
    x = s2_input()
    C_, L = S2_SHAPE
    o, sk, zap = oracle.rfi_s2(x.reshape(-1), L, C_, S2_THR)
    o = o.reshape(C_, L)
    lo, hi = oracle.sk_thresholds(L, S2_THR)
    fin = np.isfinite(sk)
    border = np.zeros(C_, bool)
    border[fin] = (np.abs(sk[fin] / hi - 1) < 1e-4) | (np.abs(sk[fin] / lo - 1) < 1e-4)
    rz = V["s2_zero_rows"]
    oz = np.all(o == 0, axis=1)
    assert np.array_equal(rz[~border], oz[~border])
    assert rz[5] and rz[9] and rz[11] and zap[11] == 0     # q5: the all-zero row was left alone, not "zapped"
    same = rz == oz
    assert np.array_equal(digests(o)[same], V["s2_rows"][same])


@pytest.mark.parametrize("C_,L,maxbox,reserve", SD_CASES)
def test_signal_detect_pipe(oracle, V, C_, L, maxbox, reserve):
    case = SD_CASES.index((C_, L, maxbox, reserve))
    f_low, bw, fs, dm, snr, chan_thr = SD_PARAMS
    x = sd_input(C_, L)
    n_input = 2 * C_ * L
    reserved = oracle.nsamps_reserved(n_input, C_, f_low, bw, fs, dm, reserve) // C_
    if reserve:
        assert reserved > 0
    res, series = oracle.signal_detect(x.reshape(-1), L, C_, reserved, snr, chan_thr, maxbox)
    assert res.detect_enabled == 1
    got = {h["boxcar"]: h for h in holders(V, f"sd_{case}")}
    exp = {int(res.boxcar_length[b]): b for b in range(res.n_boxcars) if res.signal_count[b] > 0}
    # every series the reference emits exists in the oracle with (near-)identical values and counts
    for bc, h in got.items():
        b = [i for i in range(res.n_boxcars) if res.boxcar_length[i] == bc][0]
        assert h["length"] == res.series_length[b]
        scale = np.sqrt(np.mean(h["series"].astype(np.float64) ** 2))
        assert np.abs(h["series"] - series[b, :h["length"]]).max() < 1e-4 * scale * np.sqrt(bc)
        assert abs(h["count"] - int(res.signal_count[b])) <= 1
    assert set(exp) - set(got) <= {bc for bc, b in exp.items() if res.signal_count[b] <= 1}
    assert len(got) > 0
    # the counting rule itself: the oracle's count_signal on each series the reference emitted gives the reference's
    # count, and the oracle's detector counts its own boxcar-1 series by that rule
    for h in got.values():
        assert oracle.count_signal(h["series"], snr) == h["count"]
    assert oracle.count_signal(series[0, :int(res.series_length[0])], snr) == res.signal_count[0]


@pytest.mark.parametrize("logn,C_,dm,bits", CHAIN_CASES)
def test_whole_chain_composition(oracle, V, logn, C_, dm, bits):
    """The reference's pipes composed as main.cpp:170-204 wires them (unpack -> R2C -> drop Nyquist -> s1 pipe ->
    dedisperse pipe -> waterfall FFT -> s2 pipe -> signal_detect_pipe_2), each stage being the reference's OWN code
    through the shim, against the oracle's one-call chain: pins sizes, the Nyquist drop, the [C][L] row layout, the
    normalisation coefficient and the detector's view of the spectrum — not only the stages in isolation."""
    import ctypes as CT
    import oracle_lib
    case = CHAIN_CASES.index((logn, C_, dm, bits))
    n = 1 << logn
    L = n // 2 // C_
    raw = chain_input(logn, C_, bits)
    f_low, bw, fs, avg_thr, sk_thr, snr, chan_thr, maxbox = CHAIN_PARAMS
    cfg = oracle_lib.ChainConfig()
    cfg.baseband_input_count, cfg.baseband_input_bits, cfg.window = n, bits, 0
    cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = f_low, bw, fs, dm
    cfg.baseband_reserve_sample = 0
    cfg.rfi_average_threshold, cfg.rfi_sk_threshold = avg_thr, sk_thr
    cfg.spectrum_channel_count = C_
    cfg.snr_threshold, cfg.channel_threshold, cfg.max_boxcar_length = snr, chan_thr, maxbox
    arr = (CT.c_float * 2)(1200.0, 1201.0)
    cfg.rfi_pairs, cfg.n_rfi_pairs = CT.cast(arr, CT.POINTER(CT.c_float)), 1
    work, res, series, _ = oracle.chain(raw, cfg)
    ospec = work[:n].view(np.complex64).reshape(C_, L)
    spec = V[f"chain_{case}_spectrum"]
    rz, oz = np.all(spec == 0, axis=1), np.all(ospec == 0, axis=1)
    assert (rz != oz).sum() <= 1                                  # SK border only
    same = rz == oz
    assert rel(ospec[same], spec[same]) < 2e-7                    # same arithmetic; reduction order is the runtime's
    if np.array_equal(rz, oz):
        assert res.zero_count == int(np.sum(np.abs(spec[:, 0]) ** 2 == 0))
        got = {h["boxcar"]: h for h in holders(V, f"chain_{case}")}
        for b in range(res.n_boxcars):
            bc = int(res.boxcar_length[b])
            if res.signal_count[b] > 1:
                assert bc in got and abs(got[bc]["count"] - int(res.signal_count[b])) <= 1
        for bc, h in got.items():
            b = [i for i in range(res.n_boxcars) if res.boxcar_length[i] == bc][0]
            assert h["length"] == res.series_length[b]


@pytest.mark.parametrize("nt,nf", SKV1_CASES)
def test_sk_v1(oracle, V, nt, nf):
    """alternate f-4: mitigate_rfi_spectral_kurtosis_method (v1) on the [time][frequency] layout of the refft path"""
    case = SKV1_CASES.index((nt, nf))
    x = refft_layout_block(np.random.default_rng(nt + nf), nt, nf)
    o, sk, zap = oracle.sk_v1(x.reshape(-1), nf, nt, SKV1_THR)
    o = o.reshape(nt, nf)
    lo, hi = oracle.sk_thresholds(nt, SKV1_THR)
    fin = np.isfinite(sk)
    border = np.zeros(nf, bool)
    border[fin] = (np.abs(sk[fin] / hi - 1) < 1e-4) | (np.abs(sk[fin] / lo - 1) < 1e-4)
    rz, oz = V[f"skv1_{case}_zero_cols"], np.all(o == 0, axis=0)
    assert np.array_equal(rz[~border], oz[~border])
    assert rz[5] and rz[9] and rz[11] and zap[11] == 0      # the all-zero channel is NaN -> left alone
    same = rz == oz
    # same serial fp32 sums: identical where decisions agree
    assert np.array_equal(digests(o.T)[same], V[f"skv1_{case}_cols"][same])


@pytest.mark.parametrize("nt,nf,maxbox", SDV1_CASES)
def test_signal_detect_pipe_v1(oracle, V, nt, nf, maxbox):
    """alternate f-4: the reference's signal_detect_pipe (v1: SK v1 + per-spectrum sums + boxcars) against the oracle.
    The spectrum length is a multiple of the device's work-group size here: multi_mapreduce cuts the flat array into
    pieces of ceil(size / (items * groups)) * items elements (algorithm/multi_reduce.hpp:93-101), which are the rows
    only then; the oracle restates the intended per-spectrum sum."""
    case = SDV1_CASES.index((nt, nf, maxbox))
    sk_thr, snr, chan_thr = SDV1_PARAMS
    x = refft_layout_block(np.random.default_rng(7 * nt + nf), nt, nf)
    ospec, res, series = oracle.signal_detect_v1(x.reshape(-1), nf, nt, sk_thr, snr, chan_thr, maxbox)
    assert digest(ospec) == V[f"sdv1_{case}_spectrum"]
    assert res.detect_enabled == 1 and res.zero_count == int(np.sum(np.abs(ospec.reshape(nt, nf)[0]) == 0))
    got = {h["boxcar"]: h for h in holders(V, f"sdv1_{case}")}
    exp = {int(res.boxcar_length[b]): b for b in range(res.n_boxcars) if res.signal_count[b] > 0}
    assert len(got) > 0
    for bc, h in got.items():
        b = [i for i in range(res.n_boxcars) if res.boxcar_length[i] == bc][0]
        assert h["length"] == res.series_length[b]
        if bc == 1:   # (the reference re-uses one device buffer for every boxcar > 1 and copies it asynchronously: SURVEY q3)
            scale = np.sqrt(np.mean(h["series"].astype(np.float64) ** 2))
            assert np.abs(h["series"] - series[b, :h["length"]]).max() < 1e-4 * scale
            assert abs(h["count"] - int(res.signal_count[b])) <= 1
    assert set(exp) - set(got) <= {bc for bc, b in exp.items() if res.signal_count[b] <= 1}
