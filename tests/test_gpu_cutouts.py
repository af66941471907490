"""The candidate cut-outs (srtb_b200_candidate_cutouts, Context.candidate_cutouts) on the GPU: the definition's two
bit-exact identities (the image at q = 1 is the power itself; a plane row at an incoherent trial's DM is that trial's
series), the float64 oracle (tests/cutout_oracle.py) across orientations, streams with channels masked in one stream,
decimations, widths, subbands, row counts and centres at and past both block edges, determinism, launches per call and
every refusal."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import cutout_oracle as co  # noqa: E402
import incoherent_oracle as io  # noqa: E402
import srtb_b200  # noqa: E402

E_INVALID, E_SIZE = -1, -2
SR = 2e8


def _spectra(S, C, L, seed, masked=()):
    """S random [C][L] complex64 spectra on the device; masked: (stream, channel) pairs zeroed"""
    rng = np.random.default_rng(seed)
    xs = []
    for s in range(S):
        x = (rng.standard_normal((C, L)) + 1j * rng.standard_normal((C, L))).astype(np.complex64)
        for (ms, mc) in masked:
            if ms == s:
                x[mc] = 0
        xs.append(x)
    return xs, [torch.from_numpy(x.view(np.float32)).cuda() for x in xs]


def _check(got, want, S, channels, q, where):
    tol = co.bound(S, channels, q)
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= tol * want + 1e-30), (where, float((err - tol * want).max()))


def _run_and_check(ctx, S, C, L, R, fl, bw, dm, reqs, W, nsub, n_rows, masked=(), seed=0):
    xs, d = _spectra(S, C, L, seed, masked)
    ft, dmt, rdm = ctx.candidate_cutouts(d, L, C, R, fl, bw, SR, dm, reqs, W, nsub, n_rows)
    eft, edmt, erdm = co.cutouts(xs, R, fl, bw, SR, dm, reqs, W, nsub, n_rows)
    assert np.array_equal(rdm, erdm)
    for i, r in enumerate(reqs):
        q = int(r[3])
        _check(ft[i], eft[i], S, C // nsub, q, ("ft", i, r))
        _check(dmt[i], edmt[i], S, C, q, ("dmt", i, r))
    return xs, d, ft, dmt, rdm


def test_image_at_q1_is_the_power(ctx):
    """(a): q = 1, one stream, nsub = C: ft[c][i] = |x[c][t0 + i + s]|^2 bit for bit, zero outside [0, ts)"""
    C, L, R, W = 64, 4096, 300, 256
    fl, bw, dm = 1000.0, 200.0, 30.0
    xs, d = _spectra(1, C, L, 1)
    reqs = [(1000, 31.5, 0.5, 1), (60, 29.0, 1.0, 1), (L - R - 20, 30.0, 0.0, 1)]
    ft, _, _ = ctx.candidate_cutouts(d, L, C, R, fl, bw, SR, dm, reqs, W, C, 8)
    k = co.k_table(C, fl, bw, SR)
    x = xs[0]
    p32 = (x.real * x.real + x.imag * x.imag).astype(np.float32)  # float32, no contraction
    ts = L - R
    for i, (center, d_req, _, _) in enumerate(reqs):
        s = co.shifts(k, dm, [d_req], 1)[0]
        j = center - W // 2 + np.arange(W)[None, :] + s[:, None]
        inside = (j >= 0) & (j < ts)
        want = np.where(inside, p32[np.arange(C)[:, None], np.clip(j, 0, L - 1)], np.float32(0))
        assert np.array_equal(ft[i], want), i


def test_plane_row_is_the_incoherent_series(ctx):
    """(b): q = 1, one stream, every channel kept: dmt[r][i] == v_d[t0 + i - S-] bit for bit where inside [0, T), the
    search run on the same spectrum with dms = the row DMs"""
    C, L, R, W, n_rows = 128, 8192, 500, 256, 64
    fl, bw, dm = 1200.0, -100.0, 50.0
    xs, d = _spectra(1, C, L, 2)
    reqs = [(4000, 51.0, 2.0, 1), (700, 48.5, 1.5, 1)]
    _, dmt, rdm = ctx.candidate_cutouts(d, L, C, R, fl, bw, SR, dm, reqs, W, 8, n_rows)
    for i, (center, _, _, _) in enumerate(reqs):
        dms = [float(v) for v in rdm[i]]
        h = np.zeros((srtb_b200.MAX_BOXCARS, L), np.float32)
        results, _, _, _ = ctx.incoherent_dm_search(d[0], L, C, R, fl, bw, SR, dm, dms, 1e9, 0.0, 1, h)
        # the trials' series are not handed out by the plain entry; recompute the float32 series from the definition
        # the search uses (channels in index order) through the oracle shifts, then compare the plane to it
        s, sp, sm = io.shifts(C, fl, bw, SR, dm, dms)
        assert results[0].time_series_count == L - R - sp - sm
        x = xs[0]
        p32 = (x.real * x.real + x.imag * x.imag).astype(np.float32)
        T = L - R - sp - sm
        for r in range(0, n_rows, 7):
            v = np.zeros(T, np.float32)
            for c in range(C):
                v = v + p32[c, sm + s[r, c]:sm + s[r, c] + T]
            j = center - W // 2 + np.arange(W) - sm
            inside = (j >= 0) & (j < T)
            assert np.array_equal(dmt[i, r][inside], v[j[inside]]), (i, r)


@pytest.mark.parametrize("bw", [200.0, -200.0])
@pytest.mark.parametrize("S", [1, 2, 4])
def test_against_the_oracle_streams_and_orientations(ctx, bw, S):
    C, L, R = 32, 4096, 256
    masked = [(S - 1, 5), (0, 9)] if S > 1 else [(0, 5)]
    reqs = [(1500, 41.0, 2.0, 1), (2000, 39.0, 3.0, 3), (100, 40.0, 1.0, 16), (L - R - 50, 40.5, 0.5, 1)]
    _run_and_check(ctx, S, C, L, R, 1000.0, bw, 40.0, reqs, 256, 8, 33, masked, seed=S)


@pytest.mark.parametrize("q", [1, 3, 16, 128])
def test_against_the_oracle_decimations_and_edges(ctx, q):
    """centres at, before and past both ends of [0, ts)"""
    C, L, R, W = 16, 8192, 1000, 256
    ts = L - R
    reqs = [(c, 10.0 + 0.1 * i, 1.0, q) for i, c in enumerate([0, -5, -W * q, ts - 1, ts, ts + W * q // 2, 3000])]
    _run_and_check(ctx, 2, C, L, R, 800.0, 100.0, 10.0, reqs, W, C, 4, [(1, 3)], seed=q)


@pytest.mark.parametrize("W", [2, 256, 1024])
@pytest.mark.parametrize("nsub", [1, 8, 64])
def test_against_the_oracle_widths_and_subbands(ctx, W, nsub):
    C, L, R = 64, 8192, 400
    reqs = [(3000, 60.0, 1.5, 2), (500, 61.0, 0.0, 1)]
    _run_and_check(ctx, 1, C, L, R, 1400.0, -300.0, 60.0, reqs, W, nsub, 9, seed=W + nsub)


@pytest.mark.parametrize("n_rows", [1, 2, 255, 256])
def test_against_the_oracle_row_counts(ctx, n_rows):
    C, L, R = 32, 4096, 300
    reqs = [(2000, 70.0, 4.0, 1), (1000, 72.0, 40.0, 4)]
    _, _, _, _, rdm = _run_and_check(ctx, 1, C, L, R, 1000.0, 400.0, 70.0, reqs, 256, 4, n_rows, seed=n_rows)
    if n_rows > 1:
        assert rdm[0, n_rows // 2] == np.float32(70.0)
    else:
        assert rdm[0, 0] == np.float32(70.0)


def test_config3_shape_many_requests(ctx):
    """n = 256 at config #3's stream shape (C = 2048, L = 16384), a sample of them against the oracle"""
    C, L, R, W = 2048, 16384, 1024, 256
    fl, bw, dm = 1000.0, 500.0, 100.0
    rng = np.random.default_rng(7)
    k = co.k_table(C, fl, bw, 4e9)
    xs, d = _spectra(1, C, L, 8, masked=[(0, 100), (0, 2000)])
    reqs = []
    for i in range(256):
        q = int(rng.choice([1, 2, 4, 16]))
        hw = (W // 2) * q / float(np.abs(k).max())
        reqs.append((int(rng.integers(-200, L - R + 200)), float(dm + rng.uniform(-0.05, 0.05)), hw, q))
    ft, dmt, rdm = ctx.candidate_cutouts(d, L, C, R, fl, bw, 4e9, dm, reqs, W, 256, 256)
    P = co.power(xs, R)
    for i in list(range(0, 256, 37)) + [255]:
        c, dr, hw, q = reqs[i]
        eft, edmt, erdm = co.cutout(P, k, dm, c, dr, hw, q, W, 256, 256)
        assert np.array_equal(rdm[i], erdm)
        _check(ft[i], eft, 1, C // 256, q, ("ft", i))
        _check(dmt[i], edmt, 1, C, q, ("dmt", i))


def test_two_calls_same_bytes_and_launches(ctx):
    C, L, R = 64, 4096, 100
    _, d = _spectra(2, C, L, 9)
    reqs = [(100 + 37 * i, 5.0 + 0.01 * i, 0.5, 1 + i % 5) for i in range(64)]
    n0 = ctx.launch_count
    a = ctx.candidate_cutouts(d, L, C, R, 1000.0, 200.0, SR, 5.0, reqs[:1], 256, 8, 64)
    n1 = ctx.launch_count
    b1 = ctx.candidate_cutouts(d, L, C, R, 1000.0, 200.0, SR, 5.0, reqs, 256, 8, 64)
    n2 = ctx.launch_count
    b2 = ctx.candidate_cutouts(d, L, C, R, 1000.0, 200.0, SR, 5.0, reqs, 256, 8, 64)
    assert n1 - n0 == n2 - n1 == 4
    for u, v in zip(b1, b2):
        assert u.tobytes() == v.tobytes()
    for u, v in zip(a, b1):
        assert u[0].tobytes() == v[0].tobytes()


def test_refusals(ctx):
    C, L, R = 16, 1024, 10
    _, d = _spectra(1, C, L, 10)
    ok = dict(d_spectra=d, time_count=L, chan_count=C, time_reserved_count=R, freq_low=1000.0, bandwidth=100.0,
              sample_rate=SR, dm=1.0, requests=[(500, 1.0, 0.5, 1)], width=64, nsub=4, n_rows=8)
    ctx.candidate_cutouts(**ok)
    bad_ptr = torch.zeros(2 * C * L + 2, dtype=torch.float32, device="cuda")
    nan = float("nan")
    cases = [
        (dict(d_spectra=[0]), E_INVALID),
        (dict(d_spectra=[]), E_INVALID),
        (dict(d_spectra=d * 5), E_INVALID),
        (dict(d_spectra=[bad_ptr.data_ptr() + 4]), E_INVALID),
        (dict(requests=[]), E_INVALID),
        (dict(requests=[(500, 1.0, 0.5, 1)] * 65536), E_SIZE),
        (dict(width=63), E_INVALID),
        (dict(width=0), E_SIZE),
        (dict(width=4098), E_SIZE),
        (dict(n_rows=0), E_SIZE),
        (dict(n_rows=4097), E_SIZE),
        (dict(nsub=3), E_INVALID),
        (dict(nsub=0), E_INVALID),
        (dict(requests=[(500, 1.0, 0.5, 0)]), E_INVALID),
        (dict(requests=[(500, 1.0, 0.5, (1 << 20) + 1)]), E_SIZE),
        (dict(requests=[(500, nan, 0.5, 1)]), E_INVALID),
        (dict(requests=[(500, 1.0, float("inf"), 1)]), E_INVALID),
        (dict(dm=nan), E_INVALID),
        (dict(time_reserved_count=L), E_SIZE),
        (dict(requests=[(500, 1e30, 0.5, 1)]), E_SIZE),
        (dict(requests=[(1 << 62, 1.0, 0.5, 1)]), E_SIZE),
        (dict(chan_count=0), E_INVALID),
    ]
    for change, code in cases:
        before = ctx.launch_count
        with pytest.raises(srtb_b200.SrtbError) as e:
            ctx.candidate_cutouts(**{**ok, **change})
        assert e.value.code == code, (change.keys(), e.value)
        assert ctx.launch_count == before
