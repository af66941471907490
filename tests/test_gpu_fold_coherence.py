"""The coherence products of a stream pair folded on the GPU (srtb_b200_fold_coherence, Context.fold_coherence):
random spectra against the float64 oracle (tests/fold_coherence_oracle.py) over bins, subbands, a fold_count that is no
tile multiple, a call that splits its tile ranges and channels masked in X only, in Y only and in both; agreement with
srtb_b200_fold; determinism, untouched spectra, the launch count and the argument checks; and the executable on a
seeded dual-polarisation recording whose pulse enters the second feed equal, negated and 90 degrees shifted."""
import ctypes as C
import json
import resource
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import fold_coherence_oracle as fco  # noqa: E402
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


def _pair(C_, L, seed, x_only=(3, 40), y_only=(17,), both=(29,)):
    """X and Y with channels masked in X only, in Y only and in both; x_only[0] is zero at sample 0 alone, so only the
    mask rule, not the data, keeps it out of every product"""
    rng = np.random.default_rng(seed)
    x, y = [(rng.standard_normal((C_, L)) + 1j * rng.standard_normal((C_, L))).astype(np.complex64) for _ in range(2)]
    y += (0.6 * x).astype(np.complex64)  # partly polarised, so CR and CI are far from zero
    for i, c in enumerate(x_only):
        if c < C_:
            if i == 0:
                x[c, 0] = 0
            else:
                x[c] = 0
    for c in y_only:
        if c < C_:
            y[c] = 0
    for c in both:
        if c < C_:
            x[c] = 0
            y[c] = 0
    return x, y


def _device(a):
    return torch.from_numpy(a.view(np.float32).copy()).cuda()


def _check(got, want):
    coh, hits, kept = got
    wcoh, wmag, whits, wkept = want
    assert np.array_equal(hits, whits)
    assert np.array_equal(kept, wkept)
    err = np.abs(coh - wcoh)
    assert np.all(err <= 1e-12 * wmag), float(np.max(err / np.maximum(wmag, 1e-300)))


C_, L_ = 64, 5000
PHASE = fo.phase(0.0123456, 3.2e-7, 62.5e6, 2 * C_, 987654321)  # wraps every ~96 samples, Pdot != 0


@pytest.mark.parametrize("nbin", [1, 7, 256, 4096])
@pytest.mark.parametrize("nsub", [1, 8, C_])
def test_fold_coherence_against_oracle(ctx, nbin, nsub):
    x, y = _pair(C_, L_, 300 + nbin + nsub)
    dx, dy = _device(x), _device(y)
    for F in (4321, 700):  # no tile multiple; ~1 and ~0.17 samples per bin at 4096 bins
        got = ctx.fold_coherence(dx, dy, L_, C_, F, PHASE, nbin, nsub)
        _check(got, fco.fold_coherence(x, y, F, PHASE, nbin, nsub))
        # the same hits as the plain fold of the same samples
        assert np.array_equal(got[1], ctx.fold([dx, dy], L_, C_, F, PHASE, nbin, nsub)[1])


@pytest.mark.parametrize("nsub", [1, 128])
def test_long_call_splits_tile_ranges(ctx, nsub):
    """10 tiles of 2048 samples: one tile range per tile at nsub = 1, two ranges of five tiles at nsub = C"""
    C2, L2, F = 128, 20000, 19999
    x, y = _pair(C2, L2, 11, x_only=(5, 77), y_only=(100,), both=(64,))
    got = ctx.fold_coherence(_device(x), _device(y), L2, C2, F, PHASE, 256, nsub)
    _check(got, fco.fold_coherence(x, y, F, PHASE, 256, nsub))


def test_one_sided_mask_leaves_every_product(ctx):
    """a channel masked in Y alone adds nothing to AA either: AA equals the fold of X without that channel"""
    x, y = _pair(C_, L_, 21, x_only=(), y_only=(9,), both=())
    coh, _, kept = ctx.fold_coherence(_device(x), _device(y), L_, C_, L_, PHASE, 64, 1)
    assert kept[0] == C_ - 1
    xd = x.copy()
    xd[9] = 0
    want = fo.fold([xd], L_, PHASE, 64, 1)[0][0, 0]
    assert np.allclose(coh[0, 0], want, rtol=1e-6, atol=0)
    full = fo.fold([x], L_, PHASE, 64, 1)[0][0, 0]
    assert not np.allclose(coh[0, 0], full, rtol=1e-6, atol=0)


def test_aa_bb_match_the_plain_fold(ctx):
    """without one-sided masks AA and BB are srtb_b200_fold's streams 0 and 1 (which forms |x|^2 in fp32)"""
    x, y = _pair(C_, L_, 5, x_only=(), y_only=(), both=(2, 33))
    dx, dy = _device(x), _device(y)
    for nsub, nbin in ((1, 256), (8, 7), (C_, 4096)):
        coh, hits, kept = ctx.fold_coherence(dx, dy, L_, C_, 4999, PHASE, nbin, nsub)
        prof, phits, pkept = ctx.fold([dx, dy], L_, C_, 4999, PHASE, nbin, nsub)
        assert np.array_equal(hits, phits)
        assert np.array_equal(kept, pkept[0]) and np.array_equal(kept, pkept[1])
        for p in (0, 1):
            assert np.all(np.abs(coh[p] - prof[p]) <= 1e-6 * np.abs(prof[p]))


def test_deterministic_untouched_and_three_launches(ctx):
    x, y = _pair(C_, L_, 7)
    dx, dy = _device(x), _device(y)
    bx, by = dx.clone(), dy.clone()
    for nsub, nbin in ((1, 256), (C_, 4096), (1, 1), (8, 7)):
        n0 = ctx.launch_count
        a = ctx.fold_coherence(dx, dy, L_, C_, 4999, PHASE, nbin, nsub)
        n1 = ctx.launch_count
        b = ctx.fold_coherence(dx, dy, L_, C_, 4999, PHASE, nbin, nsub)
        assert 1 <= n1 - n0 <= 3 and ctx.launch_count - n1 <= 3
        for u, v in zip(a, b):
            assert u.tobytes() == v.tobytes()
    assert torch.equal(dx, bx) and torch.equal(dy, by)


def test_bad_arguments_refused_before_any_launch(ctx):
    x, y = _pair(C_, L_, 9)
    dx, dy = _device(x), _device(y)
    lib, h = ctx.lib, ctx.h
    coh = np.zeros(4 * C_ * 4096)
    hits = np.zeros(4096, np.uint64)
    kept = np.zeros(C_, np.uint32)
    px, py = dx.data_ptr(), dy.data_ptr()

    def call(px=px, py=py, L=L_, chans=C_, F=100, phase=PHASE, nbin=16, nsub=1, out=True, hout=True, kout=True):
        return lib.srtb_b200_fold_coherence(h, px, py, L, chans, F, *phase, nbin, nsub,
                                            coh.ctypes.data if out else None, hits.ctypes.data if hout else None,
                                            kept.ctypes.data if kout else None)

    assert call() == 0
    n0 = ctx.launch_count
    assert lib.srtb_b200_fold_coherence(None, px, py, L_, C_, 100, *PHASE, 16, 1, coh.ctypes.data,
                                        hits.ctypes.data, kept.ctypes.data) == E_INVALID
    assert call(px=None) == E_INVALID
    assert call(py=None) == E_INVALID
    assert call(out=False) == E_INVALID
    assert call(hout=False) == E_INVALID
    assert call(kout=False) == E_INVALID
    assert call(L=0) == E_INVALID
    assert call(chans=0) == E_INVALID
    assert call(px=px + 4) == E_INVALID
    assert call(py=py + 4) == E_INVALID
    assert call(py=px) == E_INVALID
    assert call(F=0) == E_SIZE
    assert call(F=L_ + 1) == E_SIZE
    assert call(nbin=0) == E_SIZE
    assert call(nbin=4097) == E_SIZE
    assert call(nsub=3) == E_SIZE
    assert call(nsub=0) == E_SIZE
    assert call(chans=(1 << 24) + 64, nsub=64, L=1, F=1) == E_SIZE
    assert call(L=(1 << 40) + 1, F=(1 << 40) + 1) == E_SIZE
    assert call(phase=(float("nan"), PHASE[1], PHASE[2])) == E_INVALID
    assert call(phase=(PHASE[0], float("inf"), PHASE[2])) == E_INVALID
    assert call(phase=(PHASE[0], PHASE[1], float("-inf"))) == E_INVALID
    assert ctx.launch_count == n0
    assert "fold_coherence" in lib.srtb_b200_last_error(h).decode()


# ---- the executable on a seeded dual-polarisation recording --------------------------------------------------------
N, CH, F_LOW, BW, DM = 1 << 22, 256, 1000.0, 64.0, 1.0
SR = 2 * BW * 1e6
DT = 2 * CH / SR
PERIOD = 61.7 * DT          # not a whole number of dt
T0 = 0.3 * PERIOD           # first pulse: phase 0.3 at the top of the band
NBIN = 64


def _pulse_train(n: int, amp: float) -> np.ndarray:
    """impulses of amplitude amp at t0 + k P (arrival at the top of the band), dispersed at DM with the chirp the block
    path removes (test_gpu_fold.py's generator)"""
    R = srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)
    train = np.zeros(n, np.float64)
    t = T0
    while t * SR < n - R - 4 * CH:  # no pulse whose dispersed tail would wrap around the end
        train[int(round(t * SR))] = amp
        t += PERIOD
    f_min, bw = np.float32(F_LOW), np.float32(BW)
    f_c = float(np.float32(f_min + bw))
    spec = np.fft.rfft(train)
    f = float(f_min) + float(bw) * np.arange(spec.size, dtype=np.float64) / (n // 2)
    g = (4.148808e3 * 1e6) * float(np.float32(DM)) / f * ((f - f_c) / f_c) ** 2
    spec *= np.exp(2j * np.pi * (g - np.floor(g)))
    return np.fft.irfft(spec, n=n)


def _recording(path: Path, seed: int, amp: float, feed) -> None:
    """naocpsr_snap1, 8 bits: independent noise (sigma 20) in each polarisation, the pulse train v in stream 0 and
    feed(v) in stream 1; two samples of stream 0, then two of stream 1. The last block is short"""
    R = srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)
    n = (4 * (N - R) + N // 3) // 4 * 4
    v = _pulse_train(n, amp)
    rng = np.random.default_rng(seed)
    q = [np.clip(np.rint(rng.standard_normal(n) * 20.0 + s), -127, 127).astype(np.int8) for s in (v, feed(v))]
    raw = np.empty(2 * n, np.int8)
    raw.reshape(-1, 4)[:, 0:2] = q[0].reshape(-1, 2)
    raw.reshape(-1, 4)[:, 2:4] = q[1].reshape(-1, 2)
    raw.tofile(path)


FEEDS = {  # stream 1's pulse, and the on-pulse (CR / AA, CI / AA) it gives
    "linear": (lambda v: v, (1.0, 0.0)),
    "negated": (lambda v: -v, (-1.0, 0.0)),
    "quadrature": (lambda v: np.fft.irfft(-1j * np.fft.rfft(v), n=v.size), (0.0, 1.0)),  # rfft(y) = -i rfft(x)
}


def _run(tmp_path, name, inp, extra):
    out = tmp_path / name
    out.mkdir()
    cfg = tmp_path / f"{name}.cfg"
    cfg.write_text(f"""baseband_input_count = {N}
baseband_input_bits = -8
baseband_format_type = naocpsr_snap1
baseband_freq_low = {F_LOW}
baseband_bandwidth = {BW}
baseband_sample_rate = {SR}
baseband_reserve_sample = 1
dm = {DM}
spectrum_channel_count = {CH}
mitigate_rfi_average_method_threshold = 100
mitigate_rfi_spectral_kurtosis_threshold = 100
signal_detect_signal_noise_threshold = 7
signal_detect_max_boxcar_length = 16
input_file_path = {inp}
baseband_output_file_prefix = {out}/
fold_period = {PERIOD!r}
fold_bin_count = {NBIN}
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


def _on_pulse_ratios(out: Path):
    """(CR / AA, CI / AA) at the brightest AA bin within one of the expected bin, each product per channel-sample with
    its off-pulse median subtracted; and that bin"""
    coh = np.load(out / "fold.coherence.npy").sum(axis=0)[:, 0]          # [4][bin]
    w = np.load(out / "fold.coherence.weights.npy").sum(axis=0)[0]       # [bin]
    norm = coh / w
    want = int(np.floor((T0 / PERIOD) * NBIN))
    near = [(want + d) % NBIN for d in (-1, 0, 1)]
    off = np.ones(NBIN, bool)
    off[[(want + d) % NBIN for d in range(-3, 4)]] = False
    z = norm - np.median(norm[:, off], axis=1, keepdims=True)
    b = max(near, key=lambda i: z[0, i])
    return z[2, b] / z[0, b], z[3, b] / z[0, b], b, z[0, b] / np.std(z[0, off])


@pytest.mark.parametrize("feed", list(FEEDS))
def test_executable_folds_polarised_pulsar(tmp_path, feed):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "psr.bin"
    fn, (want_cr, want_ci) = FEEDS[feed]
    _recording(inp, 4048, 500.0, fn)
    on, err = _run(tmp_path, "on", inp, ["--fold_coherence", "1", "--fold_subintegration_blocks", "1",
                                         "--chains_per_gpu", "1"])
    assert "fold.coherence.npy" in err, err[-3000:]
    coh = np.load(on / "fold.coherence.npy")
    wts = np.load(on / "fold.coherence.weights.npy")
    assert coh.shape == (5, 4, 1, NBIN) and wts.shape == (5, 1, NBIN)
    meta = json.loads((on / "fold.json").read_text())
    assert meta["coherence"] == ["AA", "BB", "CR", "CI"] and "no calibration" in meta["coherence_definition"]
    cr, ci, b, snr = _on_pulse_ratios(on)
    assert snr > 20, (b, snr)
    assert abs(cr - want_cr) < 0.1 and abs(ci - want_ci) < 0.1, (feed, cr, ci, b, snr)
    if feed != "linear":
        return
    # the plain fold's files and the candidates do not change with the key; fold.json only gains the coherence lines
    off, _ = _run(tmp_path, "off", inp, ["--fold_subintegration_blocks", "1", "--chains_per_gpu", "1"])
    for name in ("fold.npy", "fold.weights.npy"):
        assert (on / name).read_bytes() == (off / name).read_bytes(), name
    assert _candidates(on) == _candidates(off)
    assert not list(off.glob("fold.coherence*"))
    assert "coherence" not in (off / "fold.json").read_text()
    # one chain or two: the same coherence bytes
    two, _ = _run(tmp_path, "two", inp, ["--fold_coherence", "1", "--fold_subintegration_blocks", "1",
                                         "--chains_per_gpu", "2"])
    for name in ("fold.coherence.npy", "fold.coherence.weights.npy", "fold.json"):
        assert (on / name).read_bytes() == (two / name).read_bytes(), name
