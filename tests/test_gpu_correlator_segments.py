"""The integrating, segment-averaged correlator on the H100 (srtb_b200_correlate_accumulate / _finish and the
executable's --segment_size mode) against float64 truth: every FFT plan of the segment length, every sample width,
odd and even segment counts, unbalanced input levels, long accumulations, delay recovery, alignment, launch counts,
determinism and the invalid-argument cases.

Truth is float64 torch on the device: the inputs decoded by Context.unpack (so the sample order is the library's), the
rfft of each segment, its first Ms bins, sum_s A_s conj(B_s) in float64, scaled by norm / K, and |ifft(.) Ms|.
FFT policy (as for every FFT path of the project): rel-L2 <= 1e-5 and max |error| <= 1e-4 RMS against float64."""
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import srtb_b200

ROOT = Path(__file__).resolve().parent.parent
EXE = ROOT / "src" / "srtb_b200_correlator"
E_INVALID, E_SIZE = -1, -2
BITS = [8, -8, 4, 2, 1]


def _within_policy(label, got, truth):
    got, truth = got.to(torch.float64), truth.to(torch.float64)
    rel = float(torch.linalg.vector_norm(got - truth) / torch.linalg.vector_norm(truth))
    rms = float(torch.sqrt(torch.mean(truth ** 2)))
    emax = float((got - truth).abs().max())
    print(f"{label}: rel-L2 {rel:.2e}, max-abs / RMS {emax / rms:.2e}")
    assert rel <= 1e-5, (label, rel)
    assert emax <= 1e-4 * rms, (label, emax / rms)


def _bytes(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)


def _nbytes(samples, bits):
    return samples * abs(bits) // 8


def _pair(samples, bits, seed):
    """two inputs of `samples` samples each; input 2 repeats input 1 three bytes later in one byte in 32.
    A weak correlation on purpose: a lag peak far above the rest of the output is rounded to float32 with an error of
    about eps times the peak, which exceeds 1e-4 RMS once the peak is ~1000 RMS (a fully correlated zero-mean pair at
    Ms >= 2^19 gets there), for any float32 result; one byte in 32 keeps the peak near 100 RMS."""
    n = _nbytes(samples, bits)
    a = _bytes(n + 3, seed)
    b = torch.where(_bytes(n, seed + 1) < 8, a[:n], _bytes(n, seed + 2))
    return a[3:].contiguous(), b


def _unpack(ctx, d, bits, samples):
    out = torch.empty(samples, dtype=torch.float32, device="cuda")
    ctx.unpack(d, d.numel(), bits, srtb_b200.FORMAT_SIMPLE, 0, [out], samples)
    return out


def _norm(ls):
    return float(np.float32(float(ls) ** -1.5))


def _truth(ctx, d_1, d_2, bits, ls, k):
    ms = ls // 2
    s = torch.zeros(ms, dtype=torch.complex128, device="cuda")
    step = max(1, (1 << 22) // ls)  # segments per float64 slice
    for s0 in range(0, k, step):
        n = min(step, k - s0)
        lo, hi = _nbytes(s0 * ls, bits), _nbytes((s0 + n) * ls, bits)
        x1 = _unpack(ctx, d_1[lo:hi], bits, n * ls).to(torch.float64).view(n, ls)
        x2 = _unpack(ctx, d_2[lo:hi], bits, n * ls).to(torch.float64).view(n, ls)
        s += (torch.fft.rfft(x1)[:, :ms] * torch.conj(torch.fft.rfft(x2)[:, :ms])).sum(0)
    return torch.abs(torch.fft.ifft(s * (_norm(ls) / k)) * ms)


def _segments(ctx, d_1, d_2, bits, ls, k, calls=1):
    """accumulate k segments in `calls` calls of equal size (reset on the first), then finish"""
    acc = torch.empty(ls // 2, dtype=torch.complex128, device="cuda")
    out = torch.empty(ls // 2, dtype=torch.float32, device="cuda")
    per = k // calls
    assert per * calls == k
    for c in range(calls):
        lo, hi = _nbytes(c * per * ls, bits), _nbytes((c + 1) * per * ls, bits)
        ctx.correlate_accumulate(d_1[lo:hi], d_2[lo:hi], bits, ls, per, acc, reset=c == 0)
    ctx.correlate_finish(acc, ls, k, out)
    torch.cuda.synchronize()
    return out


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _sweeps(n):
    q = n.bit_length() - 1
    return 1 if q <= 14 else 2 if q <= 20 else 3 if q <= 26 else 4


# ---- 1. agreement with whole-file mode

@pytest.mark.gpu
@pytest.mark.parametrize("n", [1 << 14, 1 << 16, 1 << 22])
def test_one_segment_equals_whole_file_mode(ctx, n):
    d_1, d_2 = _pair(n, 8, n)
    seg = _segments(ctx, d_1, d_2, 8, n, 1)
    whole = torch.empty(n // 2, dtype=torch.float32, device="cuda")
    ctx.correlate(d_1, d_2, n, whole)
    torch.cuda.synchronize()
    truth = _truth(ctx, d_1, d_2, 8, n, 1)
    _within_policy(f"segments vs correlate, {n}", seg, whole)
    _within_policy(f"segments vs truth, {n}", seg, truth)
    _within_policy(f"correlate vs truth, {n}", whole, truth)


# ---- 2. every plan and sample width

@pytest.mark.gpu
@pytest.mark.parametrize("parity", ["even", "odd"])
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("log_ls", [4, 10, 12, 13, 14, 15, 20, 22])
def test_plans_and_widths_vs_float64(ctx, log_ls, bits, parity):
    """Ls = 16 .. 2^12 (row plans), 2^13 / 2^14 (whole-row), 2^15 / 2^20 (two sweeps), 2^22 (three sweeps); about
    2^24 samples per input; an odd K leaves the last row's imaginary part zero"""
    ls = 1 << log_ls
    k = (1 << 24) // ls - (1 if parity == "odd" else 0)
    d_1, d_2 = _pair(k * ls, bits, 100 + log_ls)
    _within_policy(f"Ls 2^{log_ls} bits {bits} K {k}", _segments(ctx, d_1, d_2, bits, ls, k),
                   _truth(ctx, d_1, d_2, bits, ls, k))


# ---- 3. unbalanced amplitudes

@pytest.mark.gpu
def test_unbalanced_amplitudes(ctx):
    """input 1 full-range int8, input 2 within +-2 and correlated with it"""
    ls, k = 1 << 12, 1 << 12
    n = ls * k
    x1 = _bytes(n, 7).view(torch.int8)
    g = torch.Generator(device="cuda").manual_seed(8)
    x2 = torch.clamp(torch.round(x1.float() / 64 + torch.randn(n, device="cuda", generator=g) * 0.5), -2, 2)
    x2 = x2.to(torch.int8)
    assert float(x2.float().abs().max()) <= 2 and float(x1.float().abs().max()) >= 127
    d_1, d_2 = x1.view(torch.uint8), x2.view(torch.uint8)
    _within_policy("unbalanced", _segments(ctx, d_1, d_2, -8, ls, k), _truth(ctx, d_1, d_2, -8, ls, k))


# ---- 4. long accumulation

@pytest.mark.gpu
def test_long_accumulation(ctx):
    """K = 4096 segments of 2^12 uint8 samples, in one call and in 64 calls with reset only on the first"""
    ls, k = 1 << 12, 4096
    d_1, d_2 = _pair(ls * k, 8, 9)
    truth = _truth(ctx, d_1, d_2, 8, ls, k)
    one = _segments(ctx, d_1, d_2, 8, ls, k)
    many = _segments(ctx, d_1, d_2, 8, ls, k, calls=64)
    _within_policy("one call", one, truth)
    _within_policy("64 calls", many, truth)
    assert _bits_equal(one, _segments(ctx, d_1, d_2, 8, ls, k))
    assert _bits_equal(many, _segments(ctx, d_1, d_2, 8, ls, k, calls=64))


# ---- 5. delay recovery

def _linear_delay(stream, n, d):
    """input 1 and input 2 = input 1 delayed by d samples (not circularly): x2[t] = x1[t - d]"""
    return stream[d:d + n].contiguous(), stream[:n].contiguous()


@pytest.mark.gpu
def test_delay_recovery(ctx):
    ls, k, d = 1 << 12, 256, 100
    ms = ls // 2
    d_1, d_2 = _linear_delay(_bytes(ls * k + d, 10), ls * k, d)
    got = _segments(ctx, d_1, d_2, 8, ls, k)
    truth = _truth(ctx, d_1, d_2, 8, ls, k)
    _within_policy("delay", got, truth)
    assert int(torch.argmax(got)) == int(torch.argmax(truth)) == (-d // 2) % ms


@pytest.mark.gpu
def test_buried_delay_recovery(ctx):
    """a common int8 signal 10x below independent noise: the average over K = 1024 segments recovers the lag (the
    peak over the median at K = 1 and at K = 1024 is printed)"""
    ls, k, d = 1 << 12, 1024, 100
    n = ls * k
    g = torch.Generator(device="cuda").manual_seed(11)
    common = torch.randn(n + d, device="cuda", generator=g) * 2.0
    c_1, c_2 = _linear_delay(common, n, d)
    x1 = torch.clamp(torch.round(c_1 + torch.randn(n, device="cuda", generator=g) * 20.0), -128, 127).to(torch.int8)
    x2 = torch.clamp(torch.round(c_2 + torch.randn(n, device="cuda", generator=g) * 20.0), -128, 127).to(torch.int8)
    d_1, d_2 = x1.view(torch.uint8), x2.view(torch.uint8)
    got = _segments(ctx, d_1, d_2, -8, ls, k)
    truth = _truth(ctx, d_1, d_2, -8, ls, k)
    _within_policy("buried delay", got, truth)
    lag = (-d // 2) % (ls // 2)
    assert int(torch.argmax(got)) == int(torch.argmax(truth)) == lag
    one = _segments(ctx, d_1[:ls], d_2[:ls], -8, ls, 1)
    print(f"peak / median: K = 1 {float(one[lag] / one.median()):.1f}, K = {k} {float(got[lag] / got.median()):.1f}")


# ---- 6. alignment

@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("k", [64, 65])
def test_unaligned_inputs_bit_identical(ctx, bits, k):
    """inputs at +1 byte take the scalar unpack_one route (except 1-bit samples, whose 8-sample group is one byte):
    the same bits as aligned inputs"""
    ls = 1 << 12
    n = _nbytes(ls * k, bits)
    d_1, d_2 = _pair(ls * k, bits, 12)
    b_1, b_2 = torch.empty(n + 16, dtype=torch.uint8, device="cuda"), torch.empty(n + 16, dtype=torch.uint8,
                                                                                  device="cuda")
    b_1[1:n + 1], b_2[1:n + 1] = d_1, d_2
    aligned = _segments(ctx, d_1, d_2, bits, ls, k)
    off = _segments(ctx, b_1[1:n + 1], b_2[1:n + 1], bits, ls, k)
    assert _bits_equal(aligned, off)


# ---- 7. launch counts

@pytest.mark.gpu
@pytest.mark.parametrize("log_ls", [4, 12, 13, 14, 15, 20, 22])
def test_launch_counts(ctx, log_ls):
    """accumulate: pack + the Ls-point C2C's sweeps + split; finish: scale + the Ms-point C2C's sweeps + magnitude;
    neither depends on K"""
    ls = 1 << log_ls
    acc = torch.empty(ls // 2, dtype=torch.complex128, device="cuda")
    out = torch.empty(ls // 2, dtype=torch.float32, device="cuda")
    for k in (1, 2, 7, max(8, (1 << 23) // ls)):
        d_1, d_2 = _bytes(ls * k, 13), _bytes(ls * k, 14)
        n0 = ctx.launch_count
        ctx.correlate_accumulate(d_1, d_2, 8, ls, k, acc, reset=True)
        assert ctx.launch_count - n0 == 2 + _sweeps(ls), (ls, k)
        n0 = ctx.launch_count
        ctx.correlate_finish(acc, ls, k, out)
        assert ctx.launch_count - n0 == 2 + _sweeps(ls // 2), (ls, k)
    torch.cuda.synchronize()
    if log_ls <= 14:
        assert 2 + _sweeps(ls) == 3


# ---- 8. determinism across size changes

@pytest.mark.gpu
def test_deterministic_across_size_changes(ctx):
    cases = [(1 << 12, 300, 8, 21), (1 << 16, 33, 2, 22), (16, 5000, -8, 23), (1 << 14, 9, 4, 24), (1 << 20, 3, 1, 25)]
    inputs = [(ls, k, bits, *_pair(ls * k, bits, seed)) for ls, k, bits, seed in cases]
    first = [_segments(ctx, d_1, d_2, bits, ls, k) for ls, k, bits, d_1, d_2 in inputs]
    for _ in range(2):
        for (ls, k, bits, d_1, d_2), f in zip(inputs, first):
            assert _bits_equal(f, _segments(ctx, d_1, d_2, bits, ls, k)), (ls, k, bits)
    fresh = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        for (ls, k, bits, d_1, d_2), f in zip(reversed(inputs), reversed(first)):
            assert _bits_equal(f, _segments(fresh, d_1, d_2, bits, ls, k)), (ls, k, bits)
    finally:
        fresh.close()


# ---- 9. invalid arguments

@pytest.mark.gpu
def test_rejects_bad_arguments(ctx):
    d = _bytes(1 << 12, 15)
    acc = torch.empty(1 << 11, dtype=torch.complex128, device="cuda")
    out = torch.empty(1 << 11, dtype=torch.float32, device="cuda")
    p, pa, po = d.data_ptr(), acc.data_ptr(), out.data_ptr()
    acc_f, fin_f = ctx.lib.srtb_b200_correlate_accumulate, ctx.lib.srtb_b200_correlate_finish
    launches = ctx.launch_count
    accumulate = [((None, p, 8, 16, 1, pa, 1), E_INVALID, "null"), ((p, None, 8, 16, 1, pa, 1), E_INVALID, "null"),
                  ((p, p, 8, 16, 1, None, 1), E_INVALID, "null"), ((p, p, 8, 16, 0, pa, 1), E_INVALID, "n_segments"),
                  ((p, p, 8, 16, 1, pa + 8, 1), E_INVALID, "16-byte"), ((p, p, 8, 16, 1, pa + 4, 0), E_INVALID, "16-byte")]
    accumulate += [((p, p, b, 16, 1, pa, 1), E_INVALID, "bits") for b in (0, 3, -1, -2, -4, 16, -16, 32, 64)]
    accumulate += [((p, p, 8, ls, 1, pa, 1), E_SIZE, "power of two") for ls in (0, 1, 8, 1000, 4097, 1 << 31)]
    accumulate += [((p, p, 8, 16, (1 << 30) + 1, pa, 1), E_SIZE, "2^34"),
                   ((p, p, 8, 1 << 30, 17, pa, 0), E_SIZE, "2^34"), ((p, p, 8, 1 << 20, 1 << 40, pa, 0), E_SIZE, "2^34")]
    for args, code, text in accumulate:
        assert acc_f(ctx.h, *args) == code, args
        assert text in ctx.lib.srtb_b200_last_error(ctx.h).decode(), args
    finish = [((None, 16, 1, po), E_INVALID, "null"), ((pa, 16, 1, None), E_INVALID, "null"),
              ((pa, 16, 0, po), E_INVALID, "total_segments"), ((pa + 8, 16, 1, po), E_INVALID, "16-byte"),
              ((pa, 16, 1, po + 2), E_INVALID, "4-byte")]
    finish += [((pa, ls, 1, po), E_SIZE, "power of two") for ls in (0, 8, 1000, 1 << 31)]
    for args, code, text in finish:
        assert fin_f(ctx.h, *args) == code, args
        assert text in ctx.lib.srtb_b200_last_error(ctx.h).decode(), args
    assert ctx.launch_count == launches


# ---- 10. the executable

def _pack(samples: np.ndarray, bits: int) -> np.ndarray:
    """samples (0 .. 2^bits - 1, or int8 for -8) into bytes, sub-byte samples MSB first"""
    if abs(bits) == 8:
        return samples.astype(np.int8 if bits < 0 else np.uint8).view(np.uint8)
    per = 8 // bits
    s = samples.astype(np.uint8).reshape(-1, per)
    out = np.zeros(s.shape[0], np.uint8)
    for i in range(per):
        out |= s[:, i] << np.uint8((per - 1 - i) * bits)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bits, ls, samples_1, samples_2", [
    (8, 1 << 12, 300000, 300777),                  # sizes not powers of two
    (-8, 1 << 13, (1 << 20) + 5, 3 * (1 << 19) + 1),  # unequal sizes
    (2, 1 << 21, 70 * (1 << 21) + 4936, 70 * (1 << 21) + 800),  # 2-bit, chunks of 32, 32 and 6 segments
    (4, 1 << 16, 20 * (1 << 16) + 2, 21 * (1 << 16)),  # 4-bit, a dropped tail
])
def test_executable_equals_entries(ctx, tmp_path, bits, ls, samples_1, samples_2):
    """the output file is bit for bit the entries called with the documented chunking (max(1, 2^26 / Ls) segments per
    accumulate call, reset on the first); the stderr line reports K and the dropped samples; a known delay is found"""
    d = 200
    rng = np.random.default_rng(abs(bits) * ls)
    hi = 1 << abs(bits)
    stream = (rng.integers(-128, 128, max(samples_1, samples_2) + d) if bits == -8
              else rng.integers(0, hi, max(samples_1, samples_2) + d))
    in_1, in_2 = _pack(stream[d:d + samples_1], bits), _pack(stream[:samples_2], bits)
    in_1.tofile(tmp_path / "a.bin")
    in_2.tofile(tmp_path / "b.bin")
    r = subprocess.run([str(EXE), "--input_file_1", str(tmp_path / "a.bin"), "--input_file_2", str(tmp_path / "b.bin"),
                        "--output_file", str(tmp_path / "corr.bin"), "--segment_size", str(ls),
                        "--input_bits", str(bits)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    print(r.stderr)
    k = min(samples_1, samples_2) // ls
    assert f"K {k} segments" in r.stderr
    assert f"dropped {samples_1 - k * ls} and {samples_2 - k * ls} samples" in r.stderr
    assert samples_1 - k * ls > 0 or samples_2 - k * ls > 0
    got = torch.from_numpy(np.fromfile(tmp_path / "corr.bin", np.float32)).cuda()
    assert got.numel() == ls // 2

    d_1, d_2 = torch.from_numpy(in_1).cuda(), torch.from_numpy(in_2).cuda()
    chunk = max(1, (1 << 26) // ls)
    acc = torch.empty(ls // 2, dtype=torch.complex128, device="cuda")
    expect = torch.empty(ls // 2, dtype=torch.float32, device="cuda")
    for c, s0 in enumerate(range(0, k, chunk)):
        n = min(chunk, k - s0)
        lo, hi_ = _nbytes(s0 * ls, bits), _nbytes((s0 + n) * ls, bits)
        ctx.correlate_accumulate(d_1[lo:hi_], d_2[lo:hi_], bits, ls, n, acc, reset=c == 0)
    ctx.correlate_finish(acc, ls, k, expect)
    torch.cuda.synchronize()
    assert f"in {(k + chunk - 1) // chunk} chunks" in r.stderr
    assert _bits_equal(got, expect)
    _within_policy(f"executable bits {bits} Ls {ls}", got, _truth(ctx, d_1, d_2, bits, ls, k))
    assert int(torch.argmax(got)) == (-d // 2) % (ls // 2)
