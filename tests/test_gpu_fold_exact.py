"""The fold and the coherence fold pinned exactly at the shapes the executable folds, and the executable's fold files
pinned to a replay of its blocks.

Kernels (srtb_b200_fold, srtb_b200_fold_coherence). Spectra whose components are integers in [-64, 63]: every |x|^2
(at most 8192) is exact in fp32, every product of two components is exact, and every float64 sum is exact since the
totals stay below 2^45. So profile, hits, kept and the four coherence products must equal the float64 restatements
(tests/fold_blocks.py, which equal tests/fold_oracle.py and tests/fold_coherence_oracle.py on such spectra) bit for bit:
one lost, doubled or misbinned channel-sample fails. The shapes are the executable's: the config #3 stream shape
(C = 2048, L = 16384, one and two streams), the test recording's (C = 256, L = 8192) and a long row (C = 2048,
L = 2^16, 32 tiles), each at the fold_count a full block folds, (N - R) / 2C, and at a short last block's, with the phase
of a millisecond pulsar (Pdot != 0) far from the time origin. The launch geometry the header states (G channels per CTA,
K CTAs, R tile ranges of ntiles tiles) is computed for every case, and the cases are required to reach one tile per
range, several tiles per range with G = 64 and with G = 1, and a call without fold_finish_kernel, for both kernels.

Random spectra against float64. With u = 2^-24, each term the fold adds is t = fl32(fl32(re^2) + fl32(im^2)), so
|t - |x|^2| <= (2u + u^2) |x|^2; widening t to float64 is exact. An output adds n = (channels of the subband) x
hits[bin] non-negative terms in float64 in some order: whatever the order, the sum's error is at most
gamma_{n-1} = (n - 1) 2^-53 / (1 - (n - 1) 2^-53) times the sum. The oracle forms re^2 and im^2 exactly in float64,
rounds their sum once and adds the n terms in another order: error at most gamma_n times the exact sum. Together,
|got - want| <= (2u + u^2 + (2n + 1) 2^-53) (1 + 2^-20) want while n <= 2^32, the factor (1 + 2^-20) covering the
second-order terms (fold_blocks.fold_error_bound). The coherence products' terms are exact and may cancel; the bound
there is 1e-12 times the sum of the terms' absolute values, as in tests/test_gpu_fold_coherence.py.

Executable. src/srtb_b200 folds seeded noise recordings (tests/fold_blocks.noise_recording): 5 blocks, the last
holding 85 % of a block, so its fold count comes from the samples read; a band-limited burst that spectral kurtosis
zaps in block 2 alone, so the kept counts change from block to block; 8 subbands and 100 bins; one subintegration, or
two blocks per subintegration with a partial one at the end; one stream, and two with the coherence products; one
chain and two. The test replays each run from the documented rules alone (include/srtb_b200.h and the README):
block k starts at baseband sample k (N - R), R the reserve the reader rewinds by; its bytes are the recording's from
there, zero past the end of the file; it runs through Context.process_block with the block configuration of the .cfg;
it folds min(N - R, samples read) / 2C spectrum samples at the phase of its first sample; and the blocks' folds add in
block order, in float64, into [subint][stream][subband][bin], with weights kept x hits. The replay first requires
that the last block folds kept channels at a count the samples read set, and that some block's kept counts differ
from the block's before it. The four .npy files must equal the replay bit for bit, and fold.json its block count,
bins and subintegration starts. Each replayed block's fold is also checked against the float64 oracle on that block's spectrum."""
import json
import resource
import subprocess
import zlib
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import fold_blocks as fb  # noqa: E402
import fold_coherence_oracle as fco  # noqa: E402
import fold_oracle as fo  # noqa: E402
import srtb_b200  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent

# PSR B1937+21: about 304 spectrum samples per period at C = 2048 and 800 MHz, so a tile of 2048 holds runs of every
# length, from single samples at 4096 bins to the whole tile at one bin
PSR_P, PSR_PDOT = 0.0015578064924, 1.05e-19
FIRST_SAMPLE = (1 << 40) + 4321

# name: (N, C, freq_low, bandwidth, sample_rate, dm) of a block. The config #3 stream shape at DM 1, where the reader
# rewinds (at its own DM the smear exceeds the block and nothing is reserved); the test recording's; and a 2^28-sample
# block of the same band, whose fold_count spans 32 tiles
SHAPES = {
    "config3": (1 << 26, 2048, 1000.0, 400.0, 8e8, 1.0),
    "recording": (1 << 22, 256, 1000.0, 64.0, 128e6, 1.0),
    "long_row": (1 << 28, 2048, 1000.0, 400.0, 8e8, 1.0),
}


def _counts(shape):
    """(C, L, fold_count of a full block, fold_count of a last block holding N // 3 samples, sample rate)"""
    N, C, f_low, bw, sr, dm = SHAPES[shape]
    R = srtb_b200.nsamps_reserved(N, C, f_low, bw, sr, dm, True)
    assert 0 < R < N
    step = N - R
    return C, N // (2 * C), step // (2 * C), min(step, N // 3) // (2 * C), sr


def _cases(C):
    """(nsub, nbin) of each call: nbin 1 and 4096 at every nsub; 64 and 1024 bins at 64 subbands"""
    return [(1, 1), (1, 4096), (64, 64), (64, 1024), (C, 1), (C, 4096)]


def _device(x):
    return torch.from_numpy(x.view(np.float32)).cuda()


@pytest.fixture(scope="module")
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_launch_geometry_reaches_every_route(sm_count):
    """the cases below, with G, K, R and ntiles from the header's formulas at this device's SM count, reach one tile per
    range, several tiles per range with G = 64 and with G = 1, and a call fold_finish_kernel is skipped in, for the fold
    (4 CTAs per SM) and the coherence fold (2 per SM)"""
    table = []
    for kernel, per_sm, calls in (("fold", 4, _PLAIN), ("fold_coherence", 2, [(s, 1) for s in _COHERENCE])):
        routes = set()
        for shape, rows in calls:
            C, L, f_full, f_last, _ = _counts(shape)
            for F in (f_full, f_last):
                for nsub, nbin in _cases(C):
                    G, K, R, ntiles, finish = fb.geometry(rows, C, F, nsub, sm_count, per_sm)
                    table.append((kernel, shape, rows, F, nsub, G, K, R, ntiles, finish))
                    if R == ntiles:
                        routes.add("one tile per range")
                    if R < ntiles and G == 64:
                        routes.add("tile ranges, G = 64")
                    if R < ntiles and G == 1:
                        routes.add("tile ranges, G = 1")
                    if not finish:
                        routes.add("no finish kernel")
        assert routes == {"one tile per range", "tile ranges, G = 64", "tile ranges, G = 1", "no finish kernel"}, \
            (kernel, routes)
    print("\nkernel shape streams F nsub G K R ntiles finish")
    for row in sorted(set(table)):
        print(*row)


# ---- exact kernel cases ---------------------------------------------------------------------------------------------
_PLAIN = [("config3", 1), ("config3", 2), ("recording", 1), ("long_row", 1)]
_COHERENCE = ["config3", "recording", "long_row"]


def _phase(C, sr):
    return srtb_b200.fold_phase(PSR_P, PSR_PDOT, sr, 2 * C, FIRST_SAMPLE)


@pytest.mark.parametrize("shape,streams", _PLAIN, ids=[f"{s}-{n}streams" for s, n in _PLAIN])
def test_fold_exact_at_executable_shapes(ctx, shape, streams):
    C, L, f_full, f_last, sr = _counts(shape)
    xs = fb.integer_spectra(streams, C, L, seed=zlib.crc32(f"{shape} {streams}".encode()))
    d = [_device(x) for x in xs]
    ph = _phase(C, sr)
    assert ph[2] != 0
    for F in (f_full, f_last):
        want = fb.fold_many(xs, F, ph, _cases(C))
        for (nsub, nbin), (wprof, whits, wkept) in want.items():
            prof, hits, kept = ctx.fold(d, L, C, F, ph, nbin, nsub)
            what = (shape, streams, F, nsub, nbin)
            assert np.array_equal(hits, whits), what
            assert np.array_equal(kept, wkept), what
            assert np.array_equal(prof, wprof), (what, np.argwhere(prof != wprof)[:8])
            assert int(hits.sum()) == F and int(kept.sum()) == streams * (C - 3), what


@pytest.mark.parametrize("shape", _COHERENCE)
def test_fold_coherence_exact_at_executable_shapes(ctx, shape):
    C, L, f_full, f_last, sr = _counts(shape)
    x, y = fb.integer_spectra(2, C, L, seed=zlib.crc32(f"coherence {shape}".encode()))
    y[9] = 0                      # masked in Y alone (X's whole-row masks are Y's kept channels and vice versa)
    dx, dy = _device(x), _device(y)
    ph = _phase(C, sr)
    for F in (f_full, f_last):
        want = fb.fold_coherence_many(x, y, F, ph, _cases(C))
        for (nsub, nbin), (wcoh, _, whits, wkept) in want.items():
            coh, hits, kept = ctx.fold_coherence(dx, dy, L, C, F, ph, nbin, nsub)
            what = (shape, F, nsub, nbin)
            assert np.array_equal(hits, whits), what
            assert np.array_equal(kept, wkept), what
            assert np.array_equal(coh, wcoh), (what, np.argwhere(coh != wcoh)[:8])
            assert int(kept.sum()) == C - 7, what  # 3, 4, 5, 6, 9, C - 1 and C - 3 are masked in X or Y


# ---- random floats under the derived bound --------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fold_random_floats_within_derived_bound(ctx, shape):
    """the plain fold at every shape, the coherence fold at the two block shapes (the long row's gigabyte-class
    coherence case is the exact one above); spectra drawn channel slice by channel slice, with no full-size
    temporaries"""
    C, L, f_full, _, sr = _counts(shape)
    coherence = shape != "long_row"
    rng = np.random.default_rng(zlib.crc32(f"float {shape}".encode()))
    x, y = np.empty((C, L), np.complex64), np.empty((C, L) if coherence else (1, 1), np.complex64)
    vx, vy = x.view(np.float32).reshape(C, -1), y.view(np.float32).reshape(y.shape[0], -1)
    for c0 in range(0, C, 256):
        vx[c0:c0 + 256] = rng.standard_normal(vx[c0:c0 + 256].shape, np.float32)
        if coherence:  # partly polarised, so CR and CI do not cancel to nothing
            vy[c0:c0 + 256] = rng.standard_normal(vy[c0:c0 + 256].shape, np.float32)
            vy[c0:c0 + 256] += np.float32(0.6) * vx[c0:c0 + 256]
    x[3] = 0
    y[11 if coherence else 0] = 0
    dx, dy = _device(x), _device(y) if coherence else None
    ph = _phase(C, sr)
    worst = 0.0
    want = fb.fold_many([x], f_full, ph, _cases(C))
    for (nsub, nbin), (wprof, whits, wkept) in want.items():
        prof, hits, kept = ctx.fold([dx], L, C, f_full, ph, nbin, nsub)
        assert np.array_equal(hits, whits) and np.array_equal(kept, wkept)
        bound = fb.fold_error_bound(wprof, (C // nsub) * whits.astype(np.float64))
        err = np.abs(prof - wprof)
        assert np.all(err <= bound), (shape, nsub, nbin, float(np.max(err / np.maximum(bound, 1e-300))))
        worst = max(worst, float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0))))
    wantc = fb.fold_coherence_many(x, y, f_full, ph, _cases(C)) if coherence else {}
    for (nsub, nbin), (wcoh, wmag, whits, wkept) in wantc.items():
        coh, hits, kept = ctx.fold_coherence(dx, dy, L, C, f_full, ph, nbin, nsub)
        assert np.array_equal(hits, whits) and np.array_equal(kept, wkept)
        err = np.abs(coh - wcoh)
        assert np.all(err <= 1e-12 * wmag), (shape, nsub, nbin, float(np.max(err / np.maximum(wmag, 1e-300))))
    print(f"\n{shape}: largest err / bound of the fold {worst:.3g}")


# ---- the executable's fold files against a replay of its blocks -----------------------------------------------------
# the test recording's block: N = 2^22 samples, 256 channels over 1000-1064 MHz, DM 1; a period of 61.7 spectrum
# samples and a period derivative, 8 subbands and 100 bins
N, CH, F_LOW, BW, DM = 1 << 22, 256, 1000.0, 64.0, 1.0
SR = 2 * BW * 1e6
PERIOD = 61.7 * 2 * CH / SR
PDOT, NBIN, NSUB = 2.5e-9, 100, 8
SK = 2.0      # spectral kurtosis keeps [1, 3]: noise (2) and the short block's 85 % of data (2 / 0.85), not the burst
RFI_BLOCK, RFI_CHANNELS = 2, (100, 104)


def _recording(path, streams, seed):
    """5 blocks; the last holds 85 % of a block, more than the reader's step does not reach and no multiple of 2C,
    so its fold count is min(N - R, samples read) / 2C rounded down; block 2 alone has channels 100 to 103 zapped"""
    R = srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)
    last = (int(0.85 * N) // (4 * CH)) * (4 * CH) + 2 * 151
    assert last < N - R and last % (2 * CH)
    return fb.noise_recording(path, streams, N, R, CH, last, seed, RFI_BLOCK, RFI_CHANNELS)


def _cfg_text(fmt, inp, out, coherence):
    return f"""baseband_input_count = {N}
baseband_input_bits = -8
baseband_format_type = {fmt}
baseband_freq_low = {F_LOW}
baseband_bandwidth = {BW}
baseband_sample_rate = {SR}
baseband_reserve_sample = 1
dm = {DM}
spectrum_channel_count = {CH}
mitigate_rfi_average_method_threshold = 100
mitigate_rfi_spectral_kurtosis_threshold = {SK}
signal_detect_signal_noise_threshold = 7
signal_detect_max_boxcar_length = 16
input_file_path = {inp}
baseband_output_file_prefix = {out}/
fold_period = {PERIOD!r}
fold_period_derivative = {PDOT!r}
fold_bin_count = {NBIN}
fold_subband_count = {NSUB}
fold_coherence = {int(coherence)}
log_level = 3
"""


def _block_config(fmt):
    """the block configuration the executable builds from _cfg_text: float32 copies of the band, thresholds and dm,
    the rectangle window, the reserve on, no manual zap, no total intensity"""
    import ctypes as CT
    cfg = srtb_b200.BlockConfig()
    cfg.baseband_input_count = N
    cfg.baseband_input_bits = -8
    cfg.baseband_format = fmt
    cfg.window = srtb_b200.WINDOW_RECTANGLE
    cfg.baseband_reserve_sample = 1
    cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = F_LOW, BW, SR, DM
    cfg.mitigate_rfi_average_method_threshold = 100
    cfg.mitigate_rfi_spectral_kurtosis_threshold = SK
    cfg.spectrum_channel_count = CH
    cfg.signal_detect_signal_noise_threshold = 7
    cfg.signal_detect_channel_threshold = 0.9
    cfg.signal_detect_max_boxcar_length = 16
    cfg._keep = (CT.c_float * 1)()
    cfg.rfi_freq_pairs = CT.cast(cfg._keep, CT.POINTER(CT.c_float))
    cfg.n_rfi_freq_pairs = 0
    cfg.signal_detect_sum_streams = 0
    return cfg


def _spectrum(ptr, C, L):
    import ctypes as CT
    out = np.empty((C, L), np.complex64)
    cudart = CT.CDLL("libcudart.so")
    cudart.cudaMemcpy.argtypes = [CT.c_void_p, CT.c_void_p, CT.c_size_t, CT.c_int]
    assert cudart.cudaMemcpy(out.ctypes.data, ptr, out.nbytes, 2) == 0
    return out


def _replay(ctx, raw: bytes, fmt: int, streams: int, subint_blocks: int, coherence: bool):
    """the run's files as the documented rules make them, block by block through the library: (profile, weights,
    coherence, coherence weights, first samples of the subintegrations, blocks per subintegration, blocks), and the
    largest err / bound of the blocks' folds against float64"""
    R = srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)
    step = N - R                                   # the reader rewinds by R after every full read
    C = min(CH, N // 2)
    L = N // 2 // C
    cfg = _block_config(fmt)
    size, block_bytes = len(raw), N * streams      # 8-bit samples: one byte per sample and stream
    prof, wts, coh, cwts, starts, counts = [], [], [], [], [], []
    worst, k, blocks = 0.0, 0, []
    while True:
        first = k * step
        at = first * streams
        if at >= size:
            break
        data = raw[at:at + block_bytes]
        valid = len(data) // streams               # samples per stream the read returned
        buf = torch.zeros(block_bytes, dtype=torch.uint8).pin_memory()
        buf[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8)
        ctx.process_block(cfg, buf, block_bytes, None)
        d = [ctx.block_spectrum_ptr(s) for s in range(streams)]
        F = min(min(step, valid) // (2 * C), L)
        si = k // subint_blocks if subint_blocks else 0
        if si == len(prof):
            prof.append(np.zeros((streams, NSUB, NBIN)))
            wts.append(np.zeros((streams, NSUB, NBIN)))
            coh.append(np.zeros((4, NSUB, NBIN)))
            cwts.append(np.zeros((NSUB, NBIN)))
            starts.append(first)
            counts.append(0)
        counts[si] += 1
        blocks.append({"valid": valid, "F": F})
        if F > 0:
            ph = srtb_b200.fold_phase(PERIOD, PDOT, SR, 2 * C, first)
            p, hits, kept = ctx.fold(d, L, C, F, ph, NBIN, NSUB)
            prof[si] += p
            blocks[-1]["kept"] = kept
            wts[si] += kept.astype(np.float64)[:, :, None] * hits.astype(np.float64)[None, None, :]
            xs = [_spectrum(q, C, L) for q in d]
            wp, wh, wk = fo.fold(xs, F, ph, NBIN, NSUB)
            assert np.array_equal(hits, wh) and np.array_equal(kept, wk), k
            bound = fb.fold_error_bound(wp, (C // NSUB) * wh.astype(np.float64))
            err = np.abs(p - wp)
            assert np.all(err <= bound), (k, float(np.max(err / np.maximum(bound, 1e-300))))
            worst = max(worst, float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0))))
            if coherence:
                c, chits, ckept = ctx.fold_coherence(d[0], d[1], L, C, F, ph, NBIN, NSUB)
                assert np.array_equal(chits, hits), k
                coh[si] += c
                blocks[-1]["coherence_kept"] = ckept
                cwts[si] += ckept.astype(np.float64)[:, None] * chits.astype(np.float64)[None, :]
                wc, wm, _, wck = fco.fold_coherence(xs[0], xs[1], F, ph, NBIN, NSUB)
                assert np.array_equal(ckept, wck), k
                assert np.all(np.abs(c - wc) <= 1e-12 * wm), k
        k += 1
        if len(data) < block_bytes:                # a short read reached the end of the file: the reader stops
            break
    _check_sensitive(blocks, step, C, coherence)
    return np.stack(prof), np.stack(wts), np.stack(coh), np.stack(cwts), starts, counts, k, worst


def _check_sensitive(blocks, step, C, coherence):
    """the recording reaches what the comparison is to see: a short last block whose fold count the samples read set
    (not the step, not a whole number of spectrum samples) and which still folds kept channels, and a block whose kept
    counts differ from the block's before it"""
    last = blocks[-1]
    assert last["valid"] < step and last["F"] == last["valid"] // (2 * C) and last["valid"] % (2 * C), last
    assert last["F"] > 0 and last["kept"].sum() > 0, last
    for key in ("kept", "coherence_kept") if coherence else ("kept",):
        assert all(key in b for b in blocks), key
        assert last[key].sum() > 0, key
        changed = [k for k in range(1, len(blocks)) if not np.array_equal(blocks[k][key], blocks[k - 1][key])]
        assert RFI_BLOCK in changed, (key, [b[key].tolist() for b in blocks])


def _run(tmp_path, name, fmt_name, inp, coherence, subint_blocks, chains):
    out = tmp_path / name
    out.mkdir()
    cfg = tmp_path / f"{name}.cfg"
    cfg.write_text(_cfg_text(fmt_name, inp, out, coherence))
    exe = ROOT / "src" / "srtb_b200"
    r = subprocess.run([str(exe), "--config_file_name", str(cfg), "--fold_subintegration_blocks", str(subint_blocks),
                        "--chains_per_gpu", str(chains)], capture_output=True, text=True, timeout=600,
                       preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _check_files(out, replay, coherence, subint_blocks):
    prof, wts, coh, cwts, starts, counts, blocks, _ = replay
    names = [("fold.npy", prof), ("fold.weights.npy", wts)]
    if coherence:
        names += [("fold.coherence.npy", coh), ("fold.coherence.weights.npy", cwts)]
    for name, want in names:
        got = np.load(out / name)
        assert got.dtype == np.float64 and got.shape == want.shape, (name, got.shape, want.shape)
        bad = np.argwhere(got != want)
        assert got.tobytes() == want.tobytes(), (name, bad[:8], got[tuple(bad[0])] if len(bad) else None,
                                                 want[tuple(bad[0])] if len(bad) else None)
    meta = json.loads((out / "fold.json").read_text())
    assert meta["blocks_folded"] == blocks
    assert meta["bins"] == NBIN and meta["subbands"] == NSUB
    assert meta["blocks_per_subintegration"] == subint_blocks
    assert meta["subintegration_blocks_folded"] == counts
    assert meta["subintegration_start_s"] == [s / SR for s in starts]
    assert meta["samples_per_block_step"] == N - srtb_b200.nsamps_reserved(N, CH, F_LOW, BW, SR, DM, True)


@pytest.mark.parametrize("subint_blocks,chains", [(0, 1), (2, 2)])
def test_executable_fold_files_equal_a_replay_of_its_blocks(ctx, tmp_path, subint_blocks, chains):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "noise.bin"
    _recording(inp, 1, 2024)
    out = _run(tmp_path, "run", "simple", inp, False, subint_blocks, chains)
    replay = _replay(ctx, inp.read_bytes(), srtb_b200.FORMAT_SIMPLE, 1, subint_blocks, False)
    prof, counts, blocks = replay[0], replay[5], replay[6]
    assert blocks == 5 and prof.shape == ((1 if subint_blocks == 0 else 3), 1, NSUB, NBIN)
    assert counts == ([5] if subint_blocks == 0 else [2, 2, 1])
    _check_files(out, replay, False, subint_blocks)
    print(f"\nreplayed blocks: largest err / bound of the fold {replay[7]:.3g}")


@pytest.mark.parametrize("subint_blocks,chains", [(2, 1), (0, 2)])
def test_executable_coherence_files_equal_a_replay_of_its_blocks(ctx, tmp_path, subint_blocks, chains):
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    inp = tmp_path / "noise.bin"
    _recording(inp, 2, 4048)
    out = _run(tmp_path, "run", "naocpsr_snap1", inp, True, subint_blocks, chains)
    replay = _replay(ctx, inp.read_bytes(), srtb_b200.FORMAT_NAOCPSR_SNAP1, 2, subint_blocks, True)
    assert replay[6] == 5
    _check_files(out, replay, True, subint_blocks)
