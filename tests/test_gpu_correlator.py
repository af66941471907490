"""The baseband correlator on the H100: the cross-spectrum stage bit for bit against the oracle, srtb_b200_correlate
against float64 truth and the reference's own outputs (tests/golden/srtb_correlator_ref_vectors.npz) at every FFT plan
size it reaches, both R2C routes, odd and unequal sizes, determinism across size changes, the invalid-argument cases,
and the srtb_b200_correlator executable.

FFT policy (as for every FFT path of the project): rel-L2 <= 1e-5 and max |error| <= 1e-4 RMS against float64."""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import correlator_oracle as K
import srtb_b200

ROOT = Path(__file__).resolve().parent.parent
EXE = ROOT / "src" / "srtb_b200_correlator"
GOLDEN = Path(__file__).resolve().parent / "golden" / "srtb_correlator_ref_vectors.npz"
E_INVALID, E_SIZE = -1, -2


def _within_policy(label, got, truth):
    got = torch.as_tensor(np.asarray(got) if not torch.is_tensor(got) else got).to(torch.float64)
    truth = torch.as_tensor(np.asarray(truth) if not torch.is_tensor(truth) else truth).to(torch.float64)
    got, truth = got.to(truth.device), truth
    rel = float(torch.linalg.vector_norm(got - truth) / torch.linalg.vector_norm(truth))
    rms = float(torch.sqrt(torch.mean(truth ** 2)))
    emax = float((got - truth).abs().max())
    print(f"{label}: rel-L2 {rel:.2e}, max-abs / RMS {emax / rms:.2e}")
    assert rel <= 1e-5, (label, rel)
    assert emax <= 1e-4 * rms, (label, emax / rms)


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _correlate(ctx, d_1, d_2, input_size):
    out = torch.empty(input_size // 2, dtype=torch.float32, device="cuda")
    ctx.correlate(d_1, d_2, input_size, out)
    torch.cuda.synchronize()
    return out


def _truth_dev(d_1: torch.Tensor, d_2: torch.Tensor, input_size: int) -> torch.Tensor:
    """correlator_oracle.truth_float64 on the device (float64 torch) for inputs too long for the host"""
    m = input_size // 2
    a = torch.fft.rfft(d_1[:2 * m].to(torch.float64))[:m]
    b = torch.fft.rfft(d_2[:2 * m].to(torch.float64))[:m]
    return torch.abs(torch.fft.ifft(float(K.norm_coeff(input_size)) * a * torch.conj(b)) * m)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


# ---- cross-spectrum stage

def _complex(n, seed, off_elems=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(n + off_elems, dtype=torch.complex64, device="cuda", generator=g) * 1e3
    return base[off_elems:]


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 7, 4096, 4097, 1 << 20])
@pytest.mark.parametrize("mode", ["out_of_place", "in_place_a", "in_place_b"])
@pytest.mark.parametrize("off", [0, 1])  # complex elements: 0 = 16-byte aligned, 1 = +8 bytes
def test_cross_spectrum_bit_exact(ctx, count, mode, off):
    a, b = _complex(count, 1, off), _complex(count, 2, off)
    norm = K.norm_coeff(3 * count + 1)
    expect = K.cross_spectrum(a.cpu().numpy(), b.cpu().numpy(), norm)
    out = {"out_of_place": _complex(count, 3, off), "in_place_a": a, "in_place_b": b}[mode]
    ctx.cross_spectrum(a, b, count, float(norm), out)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), expect.view(np.uint32))


@pytest.mark.gpu
def test_cross_spectrum_mixed_alignment(ctx):
    """one input at +8 bytes takes the 8-byte route for all three pointers"""
    a, b, out = _complex(4099, 4), _complex(4099, 5, 1), _complex(4099, 6)
    norm = K.norm_coeff(12345)
    ctx.cross_spectrum(a, b, 4099, float(norm), out)
    torch.cuda.synchronize()
    expect = K.cross_spectrum(a.cpu().numpy(), b.cpu().numpy(), norm)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), expect.view(np.uint32))


@pytest.mark.gpu
def test_cross_spectrum_rejects_bad_arguments(ctx):
    a, b, out = _complex(64, 7), _complex(64, 8), _complex(64, 9)
    f = ctx.lib.srtb_b200_cross_spectrum
    pa, pb, po = a.data_ptr(), b.data_ptr(), out.data_ptr()
    launches = ctx.launch_count
    bad = [(None, pb, 64, po), (pa, None, 64, po), (pa, pb, 64, None), (pa, pb, 0, po),
           (pa + 4, pb, 8, po), (pa, pb + 4, 8, po), (pa, pb, 8, po + 4),
           (pa, pb, 64, pa + 8), (pa, pb, 64, pb - 8), (pa + 8, pb, 8, pa)]
    for d_a, d_b, n, d_o in bad:
        assert f(ctx.h, d_a, d_b, n, 1.0, d_o) == E_INVALID, (d_a, d_b, n, d_o)
    assert ctx.launch_count == launches


# ---- correlate

@pytest.mark.gpu
@pytest.mark.parametrize("name", list(K.CASES))
def test_correlate_vs_float64_and_reference(ctx, golden, name):
    """every golden pair (2 .. 2^16 bytes, 2^k + 1 sizes, unequal sizes, DC only, a known delay): float64 truth and
    the reference's own output, both within the FFT policy"""
    in_1, in_2 = K.case_inputs(name)
    input_size = min(in_1.size, in_2.size)
    got = _correlate(ctx, _dev(in_1), _dev(in_2), input_size).cpu().numpy()
    _within_policy(f"{name} vs float64", got, K.truth_float64(in_1, in_2))
    _within_policy(f"{name} vs reference", got, golden[f"{name}__out"])
    if name == "delay":
        assert int(np.argmax(got)) == int(np.argmax(golden["delay__out"]))


def _uniform_bytes(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize("input_size", [1 << 14, 1 << 15, 1 << 22, (1 << 22) + 1, 1 << 28])
def test_correlate_large_vs_float64(ctx, input_size):
    """the first raw-fused size (2^14), the whole-row C2C (2^15), three sweeps (2^22) and four sweeps (2^28)"""
    d_1, d_2 = _uniform_bytes(input_size, 11), _uniform_bytes(input_size, 12)
    got = _correlate(ctx, d_1, d_2, input_size)
    _within_policy(f"input_size {input_size}", got, _truth_dev(d_1, d_2, input_size))


@pytest.mark.gpu
@pytest.mark.parametrize("input_size", [1 << 16, 1 << 22])
def test_unpack_route_matches_truth(ctx, monkeypatch, input_size):
    """an input one byte off 16-byte alignment, and SRTB_B200_NO_FUSED_UNPACK, take the unpack kernel (one more launch
    per input) and stay within the policy"""
    d_1 = _uniform_bytes(input_size + 1, 21)
    d_2 = _uniform_bytes(input_size + 1, 22)
    truth = _truth_dev(d_1[1:], d_2[1:], input_size)
    n0 = ctx.launch_count
    fused = _correlate(ctx, d_1[1:].clone(), d_2[1:].clone(), input_size)
    n_fused = ctx.launch_count - n0
    _within_policy(f"fused {input_size}", fused, truth)

    n0 = ctx.launch_count
    off = _correlate(ctx, d_1[1:], d_2[1:], input_size)
    assert ctx.launch_count - n0 == n_fused + 2
    _within_policy(f"+1 byte {input_size}", off, truth)

    monkeypatch.setenv("SRTB_B200_NO_FUSED_UNPACK", "1")
    n0 = ctx.launch_count
    forced = _correlate(ctx, d_1[1:].clone(), d_2[1:].clone(), input_size)
    assert ctx.launch_count - n0 == n_fused + 2
    _within_policy(f"NO_FUSED_UNPACK {input_size}", forced, truth)


@pytest.mark.gpu
def test_correlate_is_deterministic_across_size_changes(ctx):
    """repeated calls give the same bits; the working buffers grow and are reused with no stale state"""
    small = [_dev(x) for x in K.case_inputs("n1k")]
    big = [_uniform_bytes(1 << 22, 31), _uniform_bytes(1 << 22, 32)]
    odd = [_uniform_bytes((1 << 16) + 1, 33), _uniform_bytes((1 << 16) + 1, 34)]
    first = [_correlate(ctx, *small, 1024), _correlate(ctx, *big, 1 << 22), _correlate(ctx, *odd, (1 << 16) + 1)]
    for _ in range(2):
        again = [_correlate(ctx, *small, 1024), _correlate(ctx, *big, 1 << 22), _correlate(ctx, *odd, (1 << 16) + 1)]
        for a, b in zip(first, again):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    fresh = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        out = torch.empty(512, dtype=torch.float32, device="cuda")
        fresh.correlate(*small, 1024, out)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), first[0].view(torch.int32))
    finally:
        fresh.close()


@pytest.mark.gpu
def test_correlate_rejects_bad_arguments(ctx):
    d = _uniform_bytes(64, 41)
    out = torch.empty(64, dtype=torch.float32, device="cuda")
    p, po = d.data_ptr(), out.data_ptr()
    f = ctx.lib.srtb_b200_correlate
    launches = ctx.launch_count
    for args, code, text in [((None, p, 64, po), E_INVALID, "null"), ((p, None, 64, po), E_INVALID, "null"),
                             ((p, p, 64, None), E_INVALID, "null"), ((p, p, 64, po + 2), E_INVALID, "aligned"),
                             ((p, p, 0, po), E_INVALID, "at least 2"), ((p, p, 1, po), E_INVALID, "at least 2"),
                             ((p, p, 6, po), E_SIZE, "[fft] n must be a power of 2"),
                             ((p, p, 7, po), E_SIZE, "[fft] n must be a power of 2"),
                             ((p, p, (1 << 31) + 2, po), E_SIZE, "[fft] n must be a power of 2"),
                             ((p, p, 1 << 32, po), E_SIZE, "2^31"), ((p, p, (1 << 32) + 1, po), E_SIZE, "2^31")]:
        assert f(ctx.h, *args) == code, args
        assert text in ctx.lib.srtb_b200_last_error(ctx.h).decode(), args
    assert ctx.launch_count == launches


# ---- the executable

def _run(args, cwd=None):
    r = subprocess.run([str(EXE), *args], cwd=cwd, capture_output=True, text=True, timeout=600)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [(1 << 16, 1 << 16), (70000, (1 << 16) + 1), ((1 << 20) + 1, 1 << 21)])
def test_executable_equals_correlate(ctx, tmp_path, sizes):
    """the output file is raw float32, bit for bit what Context.correlate gives on the same bytes (unequal and odd
    sizes: the smaller file sets input_size)"""
    rng = np.random.default_rng(sum(sizes))
    in_1, in_2 = (rng.integers(0, 256, s, dtype=np.uint8) for s in sizes)
    in_1.tofile(tmp_path / "a.bin")
    in_2.tofile(tmp_path / "b.bin")
    r = _run(["--input_file_1", str(tmp_path / "a.bin"), "--input_file_2", str(tmp_path / "b.bin"),
              "--output_file", str(tmp_path / "corr.bin"), "--gpu_device", "0"])
    assert r.returncode == 0, r.stderr
    input_size = min(sizes)
    assert f"input_size {input_size}" in r.stderr and "device" in r.stderr and "total" in r.stderr
    got = np.fromfile(tmp_path / "corr.bin", np.float32)
    expect = _correlate(ctx, _dev(in_1), _dev(in_2), input_size).cpu().numpy()
    assert got.size == input_size // 2
    assert np.array_equal(got.view(np.uint32), expect.view(np.uint32))


@pytest.mark.gpu
def test_executable_finds_a_known_delay(tmp_path):
    """input 2 is input 1 delayed by 4096 samples (circularly): the argmax is where float64 truth puts it"""
    n, delay = 1 << 20, 4096
    rng = np.random.default_rng(51)
    in_1 = rng.integers(0, 256, n, dtype=np.uint8)
    in_2 = np.roll(in_1, delay)
    in_1.tofile(tmp_path / "a.bin")
    in_2.tofile(tmp_path / "b.bin")
    r = _run(["--input_file_1", str(tmp_path / "a.bin"), "--input_file_2", str(tmp_path / "b.bin"),
              "--output_file", str(tmp_path / "corr.bin")])
    assert r.returncode == 0, r.stderr
    got = np.fromfile(tmp_path / "corr.bin", np.float32)
    truth = K.truth_float64(in_1, in_2)
    assert int(np.argmax(got)) == int(np.argmax(truth)) == (-delay // 2) % (n // 2)


@pytest.mark.gpu
def test_executable_reads_the_default_inputs(ctx, tmp_path):
    """with no input options it reads pol_1.bin and pol_2.bin in its working directory"""
    in_1, in_2 = K.case_inputs("n16k")
    in_1.tofile(tmp_path / "pol_1.bin")
    in_2.tofile(tmp_path / "pol_2.bin")
    r = _run(["--output_file", str(tmp_path / "corr.bin")], cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    got = np.fromfile(tmp_path / "corr.bin", np.float32)
    expect = _correlate(ctx, _dev(in_1), _dev(in_2), in_1.size).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), expect.view(np.uint32))
