#!/usr/bin/env python
"""Index-algebra prototype of the two-sweep config-#3 R2C that leaves its spectrum in sweep order, and of the
whole-row waterfall kernel reading its channels from that order (csrc/fft_bigrow.cuh, SRC = 1 and 2; the first
sweep is fft_col16_tma_kernel). Run on the CPU; no GPU needed.  usage: proto_r2c_sweep_order.py [logP logQ]

M = P * Q complex points packed from 2M real samples. Sweep 1 (P-point columns, stride Q) leaves
Y[k1][n2] = W_M^{k1 n2} sum_n1 x[n1 Q + n2] W_P^{n1 k1}; sweep 2 (Q-point rows) gives Z[k1][k2] = H[k1 + P k2] and
splits rows k1 and P - k1 together, so bin k = k1 + P k2 of the real transform sits at address k1 Q + k2. A channel
of L = 8 P bins is then the box of all P rows by 8 columns; the whole-row kernel's stage 0 takes chunk
d0 = 2 c + h (B1 = L / 16 = P / 2 bins) from column c, rows h P/2 ...

Checks (a) sweeps 1 + 2 + split against numpy.fft.rfft, (b) the mirror rules of the split, including the digit
complement the kernel uses for rows k1 != 0 at Q = 2^14, (c) the channel gather of stage 0 against numpy's transform
of each channel, (d) that the stage-0 reads of the sweep-order tile (16-byte pieces, lane-rotated) are conflict free
per quarter warp at P = 2^11, (e) the phase-table and zap addresses."""
import sys

import numpy as np


def sweeps(logp, logq, seed=1):
    P, Q = 1 << logp, 1 << logq
    M = P * Q
    rng = np.random.default_rng(seed)
    real = rng.standard_normal(2 * M)
    x = real[0::2] + 1j * real[1::2]
    # sweep 1: P-point DFT down each column n2, inter-sweep twiddle W_M^{k1 n2}
    cols = x.reshape(P, Q)                      # [n1][n2]
    Y = np.fft.fft(cols, axis=0)                # [k1][n2]
    k1 = np.arange(P)[:, None]
    n2 = np.arange(Q)[None, :]
    Y = Y * np.exp(-2j * np.pi * k1 * n2 / M)
    # sweep 2: Q-point DFT along each row, in place -> Z[k1][k2] = H[k1 + P k2]
    Z = np.fft.fft(Y, axis=1)
    H = np.fft.fft(x)
    kk = (np.arange(P)[:, None] + P * np.arange(Q)[None, :])
    assert np.allclose(Z, H[kk]), "sweep order"

    # split: row k1 pairs with row P - k1 (rows 0 and P/2 with themselves)
    def mirror(r, c):
        if r == 0:
            return 0, (Q - c) % Q
        if r == P // 2:
            return r, Q - 1 - c
        return P - r, Q - 1 - c

    X = np.zeros((P, Q), complex)
    for r in range(P):
        for c in range(Q):
            mr, mc = mirror(r, c)
            k = r + P * c
            assert (mr + P * mc) % M == (M - k) % M, "mirror rule"
            zk, zm = Z[r, c], np.conj(Z[mr, mc])
            w = np.exp(-1j * np.pi * k / M)
            X[r, c] = 0.5 * (zk + zm) - 0.5j * w * (zk - zm)
    ref = np.fft.rfft(real)[:M]
    err = np.abs(X.T.reshape(-1) - ref).max() / np.abs(ref).max()   # natural order: k = k1 + P k2
    assert err < 1e-12, err
    mean = np.mean(np.abs(X) ** 2)
    assert abs(mean - np.mean(np.abs(ref) ** 2)) < 1e-9 * mean
    return P, Q, M, X, ref, err


def digit_complement_ok():
    # the kernel's natural-order position of k2 (k2 = d0 + 16 d1 + 256 d2 + 4096 d3, Q = 2^14) is digit-wise, and
    # Q - 1 - k2 complements every digit: the float4 of (d3 = 2 sel, 2 sel + 1) mirrors onto (d3 = 3 - 2 sel, 2 - 2 sel),
    # the float4 at sel' = 1 - sel with its halves swapped
    Q = 1 << 14
    for k2 in range(0, Q, 4093):
        d = [k2 & 15, (k2 >> 4) & 15, (k2 >> 8) & 15, k2 >> 12]
        m = Q - 1 - k2
        assert [m & 15, (m >> 4) & 15, (m >> 8) & 15, m >> 12] == [15 - d[0], 15 - d[1], 15 - d[2], 3 - d[3]]
    return True


def channel_gather(P, Q, M, X, ref):
    L = 8 * P
    B1 = L // 16
    assert B1 == P // 2 and Q % 8 == 0
    C = M // L
    flat = X.reshape(-1)                         # address k1 Q + k2
    worst = 0.0
    for ch in range(C):
        chan = ref[ch * L:(ch + 1) * L]          # natural-order bins of the channel
        # stage 0 of the DIF transform: butterfly j over d0, inputs at row j + h B1, column 8 ch + c, d0 = 2 c + h
        stage = np.zeros((16, B1), complex)
        for j in range(B1):
            a = np.zeros(16, complex)
            for h in range(2):
                for c in range(8):
                    a[2 * c + h] = flat[(j + h * B1) * Q + 8 * ch + c]
            assert np.allclose(a, chan[j + B1 * np.arange(16)]), "chunk mapping"
            y = np.array([np.sum(a * np.exp(2j * np.pi * i * np.arange(16) / 16)) for i in range(16)])
            stage[:, j] = y * np.exp(2j * np.pi * np.arange(16) * j / L)
        # the rest of the DIF: a B1-point transform of each output chunk i gives bins i + 16 m
        out = np.zeros(L, complex)
        for i in range(16):
            out[i + 16 * np.arange(B1)] = np.fft.ifft(stage[i]) * B1
        truth = np.fft.ifft(chan) * L
        worst = max(worst, np.abs(out - truth).max() / np.abs(truth).max())
    assert worst < 1e-12, worst
    return worst


def stage0_reads_conflict_free():
    # P = 2^11: half buffer h holds rows h 1024 .. h 1024 + 1023 as [row][8] complex (64-byte rows, dense TMA boxes).
    # Thread t reads rows 2t, 2t + 1 (128 contiguous bytes) as eight 16-byte pieces; in iteration q lane t takes piece
    # q ^ (t & 7). A quarter warp (8 lanes) must touch 8 distinct 16-byte bank groups.
    NT = 512
    for q in range(8):
        for w0 in range(0, NT, 8):
            groups = {((128 * t + 16 * (q ^ (t & 7))) // 16) % 8 for t in range(w0, w0 + 8)}
            if len(groups) != 8:
                return False
    return True


def table_and_zap(P, Q, M):
    # phase table, channel-contiguous: entry ch L + 8 k1 + c holds bin k1 + P (8 ch + c); zap address of bin k
    L = 8 * P
    seen = np.zeros(M, bool)
    for idx in range(M):
        ch, r = divmod(idx, L)
        k1, c = divmod(r, 8)
        k = k1 + P * (8 * ch + c)
        assert not seen[k]
        seen[k] = True
        assert (k % P) * Q + k // P == k1 * Q + 8 * ch + c   # the spectrum address of that bin
    return bool(seen.all())


def channel_blocked_addr(k1, k2, Q):
    """address of bin k1 + P k2 in the channel-blocked layout the row sweep stores (r2c_rows_split_kernel): channel
    k2 >> 3 (L = Q = 8 P bins) is one contiguous range laid out [k1][k2 & 7]"""
    return (k2 >> 3) * Q + 8 * k1 + (k2 & 7)


def channel_blocked(P, Q, M, X, ref):
    """(a) the row sweep's outputs placed at channel_blocked_addr give every channel contiguously, in the [k1][8] order
    of stage 0's gather; (b) that order is the phase table's; (c) the manual zap's addresses of ranges across channel
    and k2' edges hit exactly the bins of the range"""
    L = 8 * P
    assert Q == L
    out = np.full(M, np.nan + 0j)
    k1 = np.arange(P)[:, None]
    k2 = np.arange(Q)[None, :]
    out[channel_blocked_addr(k1, k2, Q)] = X            # X[k1][k2] = bin k1 + P k2, as the row sweep holds it
    assert not np.isnan(out).any()
    for ch in range(M // L):
        blk = out[ch * L:(ch + 1) * L].reshape(P, 8)    # [k1][k2']: column c = bins k1 + P (8 ch + c)
        chan = ref[ch * L:(ch + 1) * L]                  # natural-order bins of the channel
        assert np.array_equal(blk, chan.reshape(8, P).T), "channel-blocked order"
    # the phase table's entry ch L + 8 k1 + c holds bin k1 + P (8 ch + c): the same address
    idx = np.arange(M)
    ch, r = idx // L, idx % L
    bins = r // 8 + P * (8 * ch + r % 8)
    assert np.array_equal(channel_blocked_addr(bins % P, bins // P, Q), idx), "phase-table order"
    # zap: ranges straddling a channel edge (bin L), a k2' edge (bin P (8 + 3)) and both (bin 2 L), as
    # rfi_zero_ranges_kernel addresses them
    logp, logq = P.bit_length() - 1, Q.bit_length() - 1
    for edge in (L, P * 11, 2 * L):
        lo, hi = edge - 3, edge + 2
        z = out.copy()
        for i in range(lo, hi + 1):
            kk1, kk2 = i & (P - 1), i >> logp
            z[((kk2 >> 3) << logq) + 8 * kk1 + (kk2 & 7)] = 0
        back = np.empty(M, complex)
        back[bins] = z                                   # natural order again
        zapped = np.nonzero(back == 0)[0]
        assert np.array_equal(zapped, np.arange(lo, hi + 1)), (edge, zapped)
        assert np.array_equal(back[:lo], ref[:lo]) and np.array_equal(back[hi + 1:], ref[hi + 1:])
    return True


def main(argv):
    logp, logq = (int(argv[1]), int(argv[2])) if len(argv) > 2 else (5, 6)
    P, Q, M, X, ref, err = sweeps(logp, logq)
    print(f"P=2^{logp} Q=2^{logq}: sweeps 1 + 2 + split vs rfft, max rel err {err:.2e}")
    assert digit_complement_ok()
    gerr = channel_gather(P, Q, M, X, ref)
    print(f"channel gather + stage 0 vs numpy: max rel err {gerr:.2e}")
    ok = stage0_reads_conflict_free()
    print("stage-0 reads conflict free:", ok)
    assert ok
    assert table_and_zap(P, Q, M)
    print("phase table / zap addresses: ok")
    return 0


def main_channel_blocked(logp=5, logq=8):
    """the channel-blocked store (Q = L = 8 P) against numpy.fft.rfft"""
    P, Q, M, X, ref, err = sweeps(logp, logq)
    X64 = X.astype(np.complex128)
    assert channel_blocked(P, Q, M, X64, X64.T.reshape(-1))
    assert np.abs(X64.T.reshape(-1) - ref).max() < 1e-12 * np.abs(ref).max()
    print(f"P=2^{logp} Q=2^{logq}: channel-blocked store, phase-table order and zap addresses: ok")
    return 0


def paired_split(logp=3, seed=2):
    """The row sweep's split at Q = L = 2^14, one read per mirror pair (r2c_rows_split_kernel). Rows k1 and P - k1 sit
    in the two CTAs of a cluster, each row in the digit-reversed layout of the whole-row kernel: Z[k2] with
    k2 = d0 + 16 d1 + 256 d2 + 4096 d3 at chunk d0 (half buffer A for d0 < 8, B for d0 >= 8), then (d1, d2, d3).
    Thread u of a CTA: lane = u & 31, wid = u >> 5, pd0 = lane & 7, h = (lane >> 3) & 1,
    pd1 = ((wid & 7) << 1) | (lane >> 4), sel = wid >> 3 (the parent's 32-bin group (pd0, pd1, sel), pd0 < 8 only).
    For j = 0..7 and i2 = h ? 15 - j : j it reads its own 16-byte pair (pd0, pd1, i2, d3 = 2 sel, 2 sel + 1) from A and
    the mirror pair (15 - pd0, 15 - pd1, 15 - i2, 1 - sel) from the mirror row's B (the partner's; its own for row P/2;
    row 0 pairs k2 with (L - k2) mod L instead and reads both from its own row), and emits X of both pairs.
    Checks: (a) every bin of every row emitted exactly once, equal to numpy.fft.rfft; (b) own reads in A, mirror reads
    in B; (c) every store instruction (a warp, one j, own or mirror pair) writes whole 64-byte pieces of the
    channel-blocked layout; (d) the fp32 partial of each 32-bin group is summed in the order i2 = 0..15 the one-group
    threads used, and the groups map one to one onto the parent's threads."""
    L = 1 << 14
    P = 1 << logp
    M = P * L
    rng = np.random.default_rng(seed)
    real = rng.standard_normal(2 * M)
    H = np.fft.fft(real[0::2] + 1j * real[1::2])
    Z = H[np.arange(P)[:, None] + P * np.arange(L)[None, :]]          # Z[k1][k2], as the row transform leaves it
    ref = np.fft.rfft(real)[:M]

    def pos(k2):  # (d0, d1, d2, d3) of natural-order k2
        return k2 & 15, (k2 >> 4) & 15, (k2 >> 8) & 15, k2 >> 12

    def split(zk, zm, k):
        zm = np.conj(zm)
        w = np.exp(-1j * np.pi * k / M)
        return 0.5 * (zk + zm) - 0.5j * w * (zk - zm)

    u = np.arange(512)
    lane, wid = u & 31, u >> 5
    pd0, h = lane & 7, (lane >> 3) & 1
    pd1, sel = ((wid & 7) << 1) | (lane >> 4), wid >> 3
    kb = pd0 + 16 * pd1 + 8192 * sel                 # own k2 of i2 = 0, d3 = 2 sel
    kbm = (15 - pd0) + 16 * (15 - pd1) + 8192 * (1 - sel)
    # the parent's thread of each group: one group per thread, bijective
    parent = lambda d0, d1, s: 32 * ((d1 >> 1) + 8 * s) + (d0 + 16 * (d1 & 1))  # noqa: E731
    assert len(set(parent(d0, d1, s) for d0 in range(16) for d1 in range(16) for s in range(2))) == 512
    # h = 1 ends with its own group's partial, h = 0 with the mirror group's: each parent thread's group exactly once
    fin = np.concatenate([parent(pd0, pd1, sel)[h == 1], parent(15 - pd0, 15 - pd1, 1 - sel)[h == 0]])
    assert np.array_equal(np.sort(fin), np.arange(512))
    # the kernel's closed forms of those two thread indices
    assert np.array_equal(parent(pd0, pd1, sel), u & ~8) and np.array_equal(parent(15 - pd0, 15 - pd1, 1 - sel), 511 - (u & ~8))
    X = np.full((P, L), np.nan + 0j)
    for i in range(P // 2):
        rows = (0, P // 2) if i == 0 else (i, P - i)
        for row in rows:
            prow = row if (row == 0 or 2 * row == P) else P - row
            for j in range(8):
                i2 = np.where(h == 1, 15 - j, j)
                im = 15 - i2
                for d3 in (0, 1):                     # the two elements of each 16-byte pair
                    k = kb + 256 * i2 + 4096 * d3                      # own bin
                    km = kbm + 256 * im + 4096 * d3                   # element d3 of the mirror pair
                    assert (pos(k)[0] < 8).all() and (pos(km)[0] >= 8).all(), "own pairs in A, mirror pairs in B"
                    if row != 0:
                        # the mirror pair holds L - 1 - k in the opposite element: no other read
                        assert np.array_equal(kbm + 256 * im + 4096 * (1 - d3), L - 1 - k)
                        mk, mkm = Z[prow, L - 1 - k], Z[row, L - 1 - km]
                    else:                             # row 0: k2 pairs with (L - k2) mod L of the same row
                        mk, mkm = Z[0, (L - k) % L], Z[0, (L - km) % L]
                    for r, kk, zk, zm in ((row, k, Z[row, k], mk), (prow, km, Z[prow, km], mkm)):
                        assert np.isnan(X[r, kk]).all(), "bin emitted twice"
                        X[r, kk] = split(zk, zm, r + P * kk)
                # (c) the store instructions of each warp: lanes 2m, 2m + 1 trade halves (own pairs: the even lane stores
                # d3 = 2 sel of k2, k2 + 1, the odd one d3 = 2 sel + 1; mirror pairs: pd0 even <-> odd swapped), so each
                # lane stores one 16-byte pair of adjacent k2 of one row
                for mine, r in ((True, row), (False, prow)):
                    base = kb if mine else kbm
                    ii = i2 if mine else im
                    odd = (pd0 & 1) if mine else 1 - (pd0 & 1)
                    ks = base - odd + 256 * ii + odd * 4096     # first k2 of the lane's 16-byte store
                    assert (ks & 1 == 0).all()
                    addr = channel_blocked_addr(r, ks, L) * 8                     # bytes
                    for w in range(16):
                        a = addr[32 * w:32 * w + 32]
                        pieces = {}
                        for x in a:
                            pieces.setdefault(x // 64, set()).add(x % 64)
                        assert all(v == {0, 16, 32, 48} for v in pieces.values()), "whole 64-byte pieces"
    assert not np.isnan(X).any(), "every bin emitted"
    err = np.abs(X.T.reshape(-1) - ref).max() / np.abs(ref).max()
    assert err < 1e-12, err
    # (d) order of the fp32 partials: h = 0 sums its own group's i2 = 0..7, h = 1 the mirror group's i2 = 0..7 (as
    # 15 - i2 descends); each keeps the other group's eight terms and folds them after the lane-8 exchange, j = 7..0
    i2_of = lambda hh, j: 15 - j if hh else j  # noqa: E731
    own = [i2_of(0, j) for j in range(8)] + [i2_of(1, j) for j in range(7, -1, -1)]
    mir = [15 - i2_of(1, j) for j in range(8)] + [15 - i2_of(0, j) for j in range(7, -1, -1)]
    assert own == list(range(16)) and mir == list(range(16))
    return err


def main_paired_split(logp=3):
    err = paired_split(logp)
    print(f"P=2^{logp} L=2^14: one read per mirror pair, both rows emitted, 64-byte store pieces, partial order: "
          f"max rel err {err:.2e}")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
