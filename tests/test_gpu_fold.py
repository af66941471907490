"""Folding at a pulsar period on the GPU (srtb_b200_fold, Context.fold): random spectra of 1, 2 and 4 streams against
the float64 oracle (tests/fold_oracle.py) over bins, subbands, a fold_count that is no tile multiple, masked channels
and both far fewer and far more than one sample per bin; determinism, untouched spectra, the launch count, the argument
checks; and the executable on a seeded recording of a periodic dispersed pulse too faint for the single-pulse detector."""
import ctypes as C
import json
import resource
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import fold_oracle as fo  # noqa: E402
import srtb_b200  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
E_INVALID, E_SIZE = -1, -2


@pytest.fixture(scope="module")
def ctx():
    torch.cuda.set_device(0)
    c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()


def _spectra(streams, C_, L, seed, zero=(3, 17, 40)):
    rng = np.random.default_rng(seed)
    out = []
    for s in range(streams):
        x = (rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64)
        for c in zero:
            if c + s < C_:
                x[c + s] = 0  # a different channel masked in each stream
        out.append(x)
    return out


def _device(xs):
    return [torch.from_numpy(x.view(np.float32).copy()).cuda() for x in xs]


def _check(got, want):
    prof, hits, kept = got
    wprof, whits, wkept = want
    assert np.array_equal(hits, whits)
    assert np.array_equal(kept, wkept)
    err = np.abs(prof - wprof)
    assert np.all(err <= 1e-5 * np.abs(wprof)), float(np.max(err / np.maximum(np.abs(wprof), 1e-300)))


C_, L_ = 64, 5000
PHASE = fo.phase(0.0123456, 3.2e-7, 62.5e6, 2 * C_, 987654321)  # wraps every ~96 samples, Pdot != 0


@pytest.mark.parametrize("streams", [1, 2, 4])
@pytest.mark.parametrize("nbin", [1, 7, 256, 4096])
@pytest.mark.parametrize("nsub", [1, 8, C_])
def test_fold_against_oracle(ctx, streams, nbin, nsub):
    xs = _spectra(streams, C_, L_, 100 + streams)
    d = _device(xs)
    for F in (4321, 700):  # ~1 and ~0.17 samples per bin at 4096 bins, hundreds at 1 and 7
        got = ctx.fold(d, L_, C_, F, PHASE, nbin, nsub)
        _check(got, fo.fold(xs, F, PHASE, nbin, nsub))


def test_bins_of_long_block_with_pdot(ctx):
    """a config #3-like row length and a phase model far from the origin: every sample's bin as the oracle has it"""
    C2, L2, F = 16, 16384, 16000
    ph = fo.phase(0.7145, 1e-12, 125e6, 2 * C2, (1 << 40) + 12345)
    xs = [np.ones((C2, L2), np.complex64)]
    prof, hits, kept = ctx.fold(_device(xs), L2, C2, F, ph, 1024, 1)
    assert np.array_equal(hits, np.bincount(fo.bins(*ph, 1024, F), minlength=1024).astype(np.uint64))
    assert np.array_equal(prof[0, 0], hits.astype(np.float64) * C2)  # |1|^2 = 1 per channel-sample, exact


def test_deterministic_untouched_and_three_launches(ctx):
    xs = _spectra(2, C_, L_, 7)
    d = _device(xs)
    before = [t.clone() for t in d]
    n0 = ctx.launch_count
    a = ctx.fold(d, L_, C_, 4999, PHASE, 256, 1)
    n1 = ctx.launch_count
    b = ctx.fold(d, L_, C_, 4999, PHASE, 256, 1)
    assert 1 <= n1 - n0 <= 3
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    for t, u in zip(d, before):
        assert torch.equal(t, u)
    for nsub, nbin in ((C_, 4096), (1, 1), (8, 7)):
        n0 = ctx.launch_count
        ctx.fold(d, L_, C_, 4999, PHASE, nbin, nsub)
        assert ctx.launch_count - n0 <= 3


def test_bad_arguments_refused_before_any_launch(ctx):
    d = _device(_spectra(1, C_, L_, 9))
    lib, h = ctx.lib, ctx.h
    prof = np.zeros(4 * C_ * 4096)
    hits = np.zeros(4096, np.uint64)
    kept = np.zeros(4 * C_, np.uint32)
    ok_ptr = d[0].data_ptr()

    def call(ptrs=(ok_ptr,), streams=1, L=L_, chans=C_, F=100, phase=PHASE, nbin=16, nsub=1, out=True):
        arr = (C.c_void_p * 4)(*(list(ptrs) + [None] * (4 - len(ptrs))))
        return lib.srtb_b200_fold(h, arr, streams, L, chans, F, *phase, nbin, nsub,
                                  prof.ctypes.data if out else None, hits.ctypes.data, kept.ctypes.data)

    n0 = ctx.launch_count
    assert call() == 0
    n0 = ctx.launch_count
    assert lib.srtb_b200_fold(h, None, 1, L_, C_, 100, *PHASE, 16, 1, prof.ctypes.data, hits.ctypes.data,
                              kept.ctypes.data) == E_INVALID
    assert call(ptrs=(None,)) == E_INVALID
    assert call(out=False) == E_INVALID
    assert call(streams=0) == E_INVALID
    assert call(ptrs=(ok_ptr,) * 4, streams=5) == E_INVALID
    assert call(ptrs=(ok_ptr + 4,)) == E_INVALID
    assert call(F=0) == E_SIZE
    assert call(F=L_ + 1) == E_SIZE
    assert call(nbin=0) == E_SIZE
    assert call(nbin=4097) == E_SIZE
    assert call(nsub=3) == E_SIZE
    assert call(nsub=0) == E_SIZE
    assert call(phase=(float("nan"), PHASE[1], PHASE[2])) == E_INVALID
    assert call(phase=(PHASE[0], float("inf"), PHASE[2])) == E_INVALID
    assert ctx.launch_count == n0
    assert "fold" in lib.srtb_b200_last_error(h).decode()


# ---- the executable on a seeded recording ------------------------------------------------------------------------
N, CH, F_LOW, BW, DM = 1 << 22, 256, 1000.0, 64.0, 1.0
SR = 2 * BW * 1e6
DT = 2 * CH / SR
PERIOD = 61.7 * DT          # not a whole number of dt
T0 = 0.3 * PERIOD           # first pulse: phase 0.3 at the top of the band
NBIN = 64


def _recording(path: Path, seed: int, amp: float) -> int:
    """8-bit single-stream noise (sigma 20) plus impulses of amplitude amp at t0 + k P (arrival at the top of the band),
    dispersed at DM with the chirp the block path removes. Returns the sample count; the last block is short"""
    R = srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)
    n = 4 * (N - R) + N // 3
    train = np.zeros(n, np.float64)
    smear = R  # no pulse whose dispersed tail would wrap around the end
    t = T0
    while t * SR < n - smear - 4 * CH:
        train[int(round(t * SR))] = amp
        t += PERIOD
    f_min, bw = np.float32(F_LOW), np.float32(BW)
    f_c = float(np.float32(f_min + bw))
    spec = np.fft.rfft(train)
    f = float(f_min) + float(bw) * np.arange(spec.size, dtype=np.float64) / (n // 2)
    g = (4.148808e3 * 1e6) * float(np.float32(DM)) / f * ((f - f_c) / f_c) ** 2
    spec *= np.exp(2j * np.pi * (g - np.floor(g)))
    v = np.fft.irfft(spec, n=n)
    del spec, train
    rng = np.random.default_rng(seed)
    q = np.clip(np.rint(rng.standard_normal(n) * 20.0 + v), -127, 127).astype(np.int8)
    q.tofile(path)
    return n


def _run(tmp_path, name, inp, extra, snr=7.0):
    out = tmp_path / name
    out.mkdir()
    cfg = tmp_path / f"{name}.cfg"
    cfg.write_text(f"""baseband_input_count = {N}
baseband_input_bits = -8
baseband_format_type = simple
baseband_freq_low = {F_LOW}
baseband_bandwidth = {BW}
baseband_sample_rate = {SR}
baseband_reserve_sample = 1
dm = {DM}
spectrum_channel_count = {CH}
mitigate_rfi_average_method_threshold = 100
mitigate_rfi_spectral_kurtosis_threshold = 1.5
signal_detect_signal_noise_threshold = {snr}
signal_detect_max_boxcar_length = 16
input_file_path = {inp}
baseband_output_file_prefix = {out}/
log_level = 3
""")
    exe = ROOT / "src" / "srtb_b200"
    r = subprocess.run([str(exe), "--config_file_name", str(cfg), *extra], capture_output=True, text=True,
                       timeout=600, preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    return out, r.stderr


def _candidates(out: Path):
    """the candidate and .tim files' contents, in block order (their names carry the wall-clock time of the read)"""
    files = sorted(p for p in out.iterdir() if not p.name.startswith(("fold", ".")))
    return [(p.name.split(".", 1)[1] if "." in p.name else "", p.read_bytes()) for p in files]


def _peak_snr(prof):
    off = np.delete(prof, np.argmax(prof))
    return int(np.argmax(prof)), (prof.max() - np.median(off)) / np.std(off)


def test_executable_folds_a_faint_pulsar(tmp_path):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "psr.bin"
    _recording(inp, 2024, amp=200.0)
    fold = ["--fold_period", repr(PERIOD), "--fold_bin_count", str(NBIN)]
    want = int(np.floor((T0 / PERIOD) * NBIN))

    # the whole run: one subintegration; no single pulse crosses the detector's threshold
    out, err = _run(tmp_path, "all", inp, fold)
    assert "folding at P" in err and "into 1 subintegration(s)" in err, err[-3000:]
    assert _candidates(out) == [], sorted(p.name for p in out.iterdir())
    prof = np.load(out / "fold.npy")
    wts = np.load(out / "fold.weights.npy")
    assert prof.shape == (1, 1, 1, NBIN) and wts.shape == prof.shape
    meta = json.loads((out / "fold.json").read_text())
    assert meta["blocks_folded"] == 5 and meta["bins"] == NBIN
    peak, snr = _peak_snr(prof[0, 0, 0] / wts[0, 0, 0])
    assert abs(peak - want) <= 1 and snr > 10, (peak, want, snr)

    # one block per subintegration: each peaks in the same bin (block timing and overlap bookkept)
    out1, _ = _run(tmp_path, "sub1", inp, fold + ["--fold_subintegration_blocks", "1", "--chains_per_gpu", "1"])
    p1 = np.load(out1 / "fold.npy") / np.load(out1 / "fold.weights.npy")
    assert p1.shape[0] == 5
    for i in range(4):  # the short last block holds too few pulses to say much
        pk, s = _peak_snr(p1[i, 0, 0])
        assert abs(pk - want) <= 1, (i, pk, want, s)
    assert json.loads((out1 / "fold.json").read_text())["subintegration_start_s"][1] > 0

    # one chain or two: the same bytes
    out2, _ = _run(tmp_path, "sub2", inp, fold + ["--fold_subintegration_blocks", "1", "--chains_per_gpu", "2"])
    for name in ("fold.npy", "fold.weights.npy", "fold.json"):
        assert (out1 / name).read_bytes() == (out2 / name).read_bytes(), name


def test_executable_candidates_unchanged_by_folding(tmp_path):
    """at a threshold the periodic pulses cross, the candidate and .tim files are the same with folding on and off"""
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "psr.bin"
    _recording(inp, 2024, amp=200.0)
    off, _ = _run(tmp_path, "off", inp, ["--chains_per_gpu", "1"], snr=2.5)
    on, _ = _run(tmp_path, "on", inp, ["--chains_per_gpu", "1", "--fold_period", repr(PERIOD)], snr=2.5)
    a, b = _candidates(off), _candidates(on)
    assert a and a == b
    assert not list(off.glob("fold*")) and (on / "fold.npy").exists()
