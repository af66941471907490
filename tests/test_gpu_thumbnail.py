"""srtb_b200_simplify_spectrum (the waterfall thumbnail of simplify_spectrum_pipe_2) on the GPU against the CPU
oracle (tests/thumbnail_oracle.py, itself pinned bit for bit to the reference by test_thumbnail_oracle.py), and the
executable's waterfall PPM.

Tolerances: the intensities are sums of at most a few hundred positive fp32 terms, taken in another order than the
reference's work-item split: rel-L2 <= 1e-6 and per pixel <= 1e-5 relative. The device average is a fixed-order tree
over all pixels, more accurate than the reference's serial partial sums, so it is held to 1e-6 of the exact (float64)
mean of the oracle's intensities and to 1e-5 of the oracle's own fp32 average. Pixmaps are equal except on pixels whose
oracle intensity lies within 1e-5 relative of a colour-channel step or of 1 (the borderline rule of the parity tests;
the alpha channel, 255 at both ends of the colour range, is on a step for every intensity); each differing pixel must be
such a pixel, and their number is reported."""
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import thumbnail_oracle as T

ROOT = Path(__file__).resolve().parent.parent
E_INVALID = -1


@pytest.fixture(scope="module")
def env():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import srtb_b200
    torch.cuda.set_device(0)
    ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield torch, srtb_b200, ctx
    ctx.close()


def _run(env, d_spec, L, C, W, H):
    torch, _, ctx = env
    inten = torch.empty((H, W), dtype=torch.float32, device="cuda")
    pix = torch.empty((H, W), dtype=torch.int32, device="cuda")
    avg = torch.empty(1, dtype=torch.float32, device="cuda")
    ctx.simplify_spectrum(d_spec, L, C, W, H, inten, pix, avg)
    torch.cuda.synchronize()
    return inten.cpu().numpy(), pix.cpu().numpy().view(np.uint32), avg.cpu().numpy()[0]


def _check(label, got, ref):
    inten, pix, avg = got
    raw, ravg, rinten, rpix = ref
    exact_mean = np.mean(raw, dtype=np.float64)
    assert abs(float(avg) - exact_mean) <= 1e-6 * exact_mean, (label, float(avg), exact_mean)
    assert abs(float(avg) - float(ravg)) <= 1e-5 * float(ravg), (label, float(avg), float(ravg))
    r64 = rinten.astype(np.float64)
    rel_l2 = np.linalg.norm(inten - r64) / max(np.linalg.norm(r64), 1e-300)
    assert rel_l2 <= 1e-6, (label, rel_l2)
    per = np.abs(inten - r64) / np.maximum(np.abs(r64), 1e-300)
    per[(inten == 0) & (rinten == 0)] = 0
    assert per.max() <= 1e-5, (label, per.max(), np.unravel_index(per.argmax(), per.shape))
    ndiff, nbad = T.unexplained_pixels(rinten, rpix, pix)
    assert nbad == 0, (label, nbad, ndiff)
    print(f"{label}: rel-L2 {rel_l2:.2e}, max per-pixel {per.max():.2e}, average {float(avg):.6g} "
          f"(oracle {float(ravg):.6g}), borderline pixels differing {ndiff} of {pix.size}")
    return ndiff


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(T.CASES))
def test_thumbnail_matches_oracle(env, name):
    torch = env[0]
    C, L, H, W, _ = T.CASES[name]
    spec = T.case_spectrum(name)
    got = _run(env, torch.from_numpy(spec).cuda(), L, C, W, H)
    _check(name, got, T.simplify_spectrum(spec, W, H))


@pytest.mark.gpu
@pytest.mark.parametrize("C,L,H,W,offset", [(30, 333, 20, 45, 0),      # odd row length: 8-byte loads
                                            (64, 1000, 24, 70, 1),     # spectrum not 16-byte aligned
                                            (7, 5, 33, 41, 0)])        # upsampling both axes far (q12 everywhere)
def test_thumbnail_load_paths(env, C, L, H, W, offset):
    torch = env[0]
    rng = np.random.default_rng(C * L)
    spec = (rng.standard_normal((C, L)) + 1j * rng.standard_normal((C, L))).astype(np.complex64)
    buf = torch.zeros(C * L + offset, dtype=torch.complex64, device="cuda")
    buf[offset:] = torch.from_numpy(spec.ravel()).cuda()
    got = _run(env, buf.data_ptr() + 8 * offset, L, C, W, H)
    _check(f"{C}x{L}->{H}x{W}+{offset}", got, T.simplify_spectrum(spec, W, H))


def _block_cfg(srtb_b200, n, chans):
    cfg = srtb_b200.BlockConfig()
    cfg.baseband_input_count, cfg.baseband_input_bits = n, -8
    cfg.baseband_format, cfg.window, cfg.baseband_reserve_sample = srtb_b200.FORMAT_SIMPLE, 0, 0
    cfg.baseband_freq_low, cfg.baseband_bandwidth, cfg.baseband_sample_rate, cfg.dm = 1000.0, 400.0, 8e8, 562.05
    cfg.mitigate_rfi_average_method_threshold = 10.0
    cfg.mitigate_rfi_spectral_kurtosis_threshold = 1.1
    cfg.spectrum_channel_count = chans
    cfg.signal_detect_signal_noise_threshold = 6.0
    cfg.signal_detect_channel_threshold = 0.9
    cfg.signal_detect_max_boxcar_length = 64
    cfg.n_rfi_freq_pairs = 0
    return cfg


@pytest.mark.gpu
def test_thumbnail_of_a_config3_block(env):
    """a real block's dynamic spectrum (2^26 samples, 2048 channels: [2048][16384]) -> 1080 x 1920"""
    torch, srtb_b200, ctx = env
    n, C = 1 << 26, 2048
    L = n // 2 // C
    rng = np.random.default_rng(3)
    v = rng.standard_normal(n, dtype=np.float32) * 20
    v[n // 3:n // 3 + 4096] += rng.standard_normal(4096, dtype=np.float32) * 90
    bb = np.clip(np.round(v), -127, 127).astype(np.int8)
    h_series = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
    ctx.process_block(_block_cfg(srtb_b200, n, C), torch.from_numpy(bb.view(np.uint8)).pin_memory(), n, h_series)
    d_spec = ctx.block_spectrum_ptr(0)
    got = _run(env, d_spec, L, C, 1920, 1080)
    spec = torch.empty(C * L, dtype=torch.complex64, device="cuda")
    ctx.synchronize()
    import ctypes as CT
    cudart = CT.CDLL("libcudart.so")
    cudart.cudaMemcpy.argtypes = [CT.c_void_p, CT.c_void_p, CT.c_size_t, CT.c_int]
    assert cudart.cudaMemcpy(spec.data_ptr(), d_spec, C * L * 8, 3) == 0
    h = spec.cpu().numpy().reshape(C, L)
    assert np.count_nonzero(np.all(h == 0, axis=1)) < C  # not an all-zapped block
    _check("config3 block", got, T.simplify_spectrum(h, 1920, 1080))


@pytest.mark.gpu
def test_thumbnail_of_config1_rows(env):
    """[2048][2^18] (config #1's rows) -> 1080 x 1920: 137 input cells per pixel along time. |x|^2 for the oracle is
    taken elementwise (re * re + im * im, one rounding each) on the device, to keep 4 GiB of spectrum off the host."""
    torch = env[0]
    C, L = 2048, 1 << 18
    g = torch.Generator(device="cuda").manual_seed(1)
    spec = torch.randn(C, L, dtype=torch.complex64, device="cuda", generator=g)
    spec[100:140] = 0
    got = _run(env, spec, L, C, 1920, 1080)
    re, im = spec.real, spec.imag
    p = torch.add(torch.mul(re, re), torch.mul(im, im)).cpu().numpy()
    del spec, re, im
    _check("config1 rows", got, T.simplify_spectrum(p, 1920, 1080))


@pytest.mark.gpu
def test_thumbnail_is_deterministic_and_survives_resizes(env):
    torch, _, ctx = env
    specs = {}
    for name in ("nonint_wide", "upsample", "wide_ratio"):
        specs[name] = torch.from_numpy(T.case_spectrum(name)).cuda()

    def call(name):
        C, L, H, W, _ = T.CASES[name]
        return _run(env, specs[name], L, C, W, H)

    first = {k: call(k) for k in specs}
    launches = ctx.launch_count
    for name in ("upsample", "nonint_wide", "wide_ratio", "nonint_wide"):  # scratch grows, shrinks, grows
        again = call(name)
        for a, b in zip(first[name], again):
            assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), name
    assert ctx.launch_count - launches == 3 * 4


@pytest.mark.gpu
def test_thumbnail_rejects_bad_arguments(env):
    torch, srtb_b200, ctx = env
    lib, h = ctx.lib, ctx.h
    spec = torch.zeros(64, dtype=torch.complex64, device="cuda")
    inten = torch.empty(16, dtype=torch.float32, device="cuda")
    pix = torch.empty(16, dtype=torch.int32, device="cuda")
    launches = ctx.launch_count
    s, i, p = spec.data_ptr(), inten.data_ptr(), pix.data_ptr()
    c0, c1, co = srtb_b200.GUI_COLOR_0, srtb_b200.GUI_COLOR_1, srtb_b200.GUI_COLOR_OVERFLOW
    bad = [(h, None, 8, 8, 4, 4, i, p), (h, s, 8, 8, 4, 4, None, p), (h, s, 8, 8, 4, 4, i, None),
           (h, s, 0, 8, 4, 4, i, p), (h, s, 8, 0, 4, 4, i, p), (h, s, 8, 8, 0, 4, i, p), (h, s, 8, 8, 4, 0, i, p),
           (None, s, 8, 8, 4, 4, i, p)]
    for hh, ss, L, C, W, H, ii, pp in bad:
        assert lib.srtb_b200_simplify_spectrum(hh, ss, L, C, W, H, c0, c1, co, ii, pp, None) == E_INVALID
    assert ctx.launch_count == launches


def _replay(tmp_path, gui: int, width: int = 200, height: int = 48):
    exe = ROOT / "src" / "srtb_b200"
    subprocess.run(["make", "-C", str(ROOT / "src")], check=True, capture_output=True)
    logn, C_ = 18, 64
    n = 1 << logn
    blocks = []
    for seed in range(71, 74):
        rng = np.random.default_rng(seed)
        v = rng.standard_normal(n) * 20
        v += 40 * np.cos(2 * np.pi * 0.1185 * np.arange(n))
        v[n // 2:n // 2 + 256] += rng.standard_normal(256) * 110
        blocks.append(np.clip(np.round(v), -127, 127).astype(np.int8))
    inp = tmp_path / "bb.bin"
    np.concatenate(blocks).tofile(inp)
    prefix = tmp_path / "cand_"
    cfg = tmp_path / "replay.cfg"
    cfg.write_text(f"""# replay with the waterfall thumbnail
baseband_input_count = 2 ** {logn}
baseband_input_bits = -8
baseband_format_type = simple
baseband_freq_low = 1000.0
baseband_bandwidth = 500.0
baseband_sample_rate = 1000 * 1e6
baseband_reserve_sample = 0
dm = 0
spectrum_channel_count = 2 ** 6
mitigate_rfi_average_method_threshold = 5
mitigate_rfi_spectral_kurtosis_threshold = 1.3
signal_detect_signal_noise_threshold = 6
signal_detect_max_boxcar_length = 64
input_file_path = {inp}
baseband_output_file_prefix = {prefix}
gui_enable = {gui}
gui_pixmap_width = {width}
gui_pixmap_height = {height}
log_level = 2
""")
    return subprocess.run([str(exe), "--config_file_name", str(cfg), "--chains_per_gpu", "2", "--ring_depth", "3"],
                          capture_output=True, text=True, timeout=600), C_, n // 2 // C_


def _read_ppm(path):
    data = path.read_bytes()
    m = re.match(rb"P6\n(\d+) (\d+)\n255\n", data)
    assert m, data[:32]
    w, h = int(m.group(1)), int(m.group(2))
    rgb = np.frombuffer(data[m.end():], np.uint8)
    assert rgb.size == w * h * 3
    return rgb.reshape(h, w, 3)


@pytest.mark.gpu
def test_executable_writes_the_waterfall(tmp_path):
    r, C_, L = _replay(tmp_path, gui=1)
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"waterfall: (\d+) thumbnail\(s\) written, (\d+) block\(s\) skipped", r.stderr)
    assert m and int(m.group(1)) >= 1 and int(m.group(1)) + int(m.group(2)) == 3, r.stderr[-2000:]
    ppm = tmp_path / "cand_waterfall.0.ppm"
    assert ppm.exists(), sorted(p.name for p in tmp_path.iterdir())
    assert not list(tmp_path.glob("*.tmp"))
    img = _read_ppm(ppm)
    assert img.shape == (48, 200, 3)
    # every block has a burst, so every block's spectrum is in a candidate .npy: the image is one of theirs
    npys = sorted(tmp_path.glob("cand_*.npy"))
    assert len(npys) == 3
    ok = []
    for p in npys:
        spec = np.load(p)
        assert spec.shape == (C_, L)
        _, _, rinten, rpix = T.simplify_spectrum(spec, 200, 48)
        got = (np.uint32(T.COLOR_0) & np.uint32(0xFF000000)) | (img[..., 0].astype(np.uint32) << 16) | \
            (img[..., 1].astype(np.uint32) << 8) | img[..., 2].astype(np.uint32)  # alpha is not in the file
        ndiff, nbad = T.unexplained_pixels(rinten, rpix | np.uint32(0xFF000000), got)
        if nbad == 0:
            ok.append((p.name, ndiff))
    assert ok, "the waterfall matches none of the replayed blocks"
    print(f"waterfall.0.ppm matches {ok}")


@pytest.mark.gpu
def test_executable_without_gui_writes_no_waterfall(tmp_path):
    r, _, _ = _replay(tmp_path, gui=0)
    assert r.returncode == 0, r.stderr[-2000:]
    assert list(tmp_path.glob("cand_*.npy"))
    assert not list(tmp_path.glob("*.ppm*"))


def test_executable_rejects_an_empty_pixmap(tmp_path):
    """gui_enable with a zero gui_pixmap_width or gui_pixmap_height stops at start-up, before any device is touched"""
    exe = ROOT / "src" / "srtb_b200"
    if not exe.exists():
        pytest.skip("src/srtb_b200 not built")
    for w, h in [(0, 48), (200, 0)]:
        cfg = tmp_path / "bad.cfg"
        cfg.write_text(f"gui_enable = 1\ngui_pixmap_width = {w}\ngui_pixmap_height = {h}\n")
        r = subprocess.run([str(exe), "--config_file_name", str(cfg)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2 and "gui_pixmap" in r.stderr, (r.returncode, r.stderr[-500:])
