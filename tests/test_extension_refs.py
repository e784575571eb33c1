"""Plain references for the two kernels the reference project does not implement, written from their definitions in
numpy / Python and sharing no code with oracle/sr_oracle.c (whose restatements sro_dtw_band and sro_mfcc_geom_b read the
same generated tables as the kernels, so a mistake common to both would pass every parity test):

  K3  the Sakoe-Chiba banded DP (dtw_band_kernel for r != 10, dtw_band_thread_kernel<10>): band_dp_ref of refs.py,
      itself checked against a textbook full-matrix DTW where the band covers every column and against the closed form
      of r = 0;
  K5  the GEOM_B front end (mfcc_geomb_kernel): its tables from the float64 formulas, and the 256-point FFT (the oracle's
      cr4_fft_generic.c on the CPU, the shared core's fft_radix4<256> on the device) against the exact DFT / N.

CPU tests pin the oracle to these references, so that the GPU tests and `bench.py --workload dtw_band | mfcc_b`, which
compare the kernels with the oracle, rest on a checked checker."""
import os

import numpy as np
import pytest

import oracle_bind as ob
import sr_b200
from cases import band_cases, band_rows, guard_edge_shapes, make_ftr
from refs import (DIS_ERR, MAX_A, MAX_B, MAX_FRM, NTHREADS, band_dp_ref, dist_matrix, full_dp_ref, guard_rejects)


# ---- references --------------------------------------------------------------------------------------------------
def band0_closed_form(fin, fmdl):
    """r = 0: row i holds only the cell (i, floor(i*M/I)), so the one possible path is those cells; it exists when every
    row-to-row shift is at most 1 (an up or a diagonal step) and the last row's cell is column M-1"""
    I, M = len(fin), len(fmdl)
    if guard_rejects(I, M):
        return DIS_ERR
    cols = [i * M // I for i in range(I)]
    if cols[-1] != M - 1 or any(b - a > 1 for a, b in zip(cols, cols[1:])):
        return DIS_ERR
    d = dist_matrix(fin, fmdl)
    return int(sum(int(d[i, c]) for i, c in enumerate(cols))) // (I + M)


def dft_over_n(re, im):
    """the exact DFT / N of each row, in float64"""
    N = re.shape[1]
    return np.fft.fft(re.astype(np.float64) + 1j * im.astype(np.float64), axis=1) / N


# ---- K3 on the CPU: the reference against band-free references, then the oracle against the reference ------------
def test_dist_matrix_is_get_dis():
    """dist_matrix is the reference's get_dis element for element (the reference's own C when it is built), at the
    rounding corners: sums that wrap, that round up to 2^32 in float32 (d = 65 536), and perfect squares +- 1"""
    rng = np.random.default_rng(45)
    a = rng.integers(-32768, 32768, (600, 12)).astype(np.int16)
    b = rng.integers(-32768, 32768, (600, 12)).astype(np.int16)
    a[:100] = rng.integers(-3000, 3001, (100, 12))
    b[:100] = a[:100]
    b[:100, 0] += rng.integers(-2, 3, 100).astype(np.int16)
    a[100], b[100] = MAX_A, MAX_B
    a[101], b[101] = (32767,) * 12, (-32767,) * 12
    want = ob.best_oracle().get_dis(a, b)
    got = np.array([dist_matrix(a[i:i + 1], b[i:i + 1])[0, 0] for i in range(len(a))], np.uint32)
    assert np.array_equal(got, want)
    assert got[100] == 65536 and got[101] == 65511


def test_band_dp_ref_equals_full_dp_and_the_r0_closed_form():
    """band_dp_ref against two references with no band logic: for M <= r + 1 the band covers every column of every row
    (c in [0, M-1]), so the banded result is the full DP's; for r = 0 it is the closed form (with M = I: the diagonal sum
    over 2I). Shapes: both sides of the guard edges up to 24 rows, every kind of input"""
    rng = np.random.default_rng(3)
    shapes = [(I, M) for I in range(1, 25) for M in range(1, 25) if I <= 2 * M + 1 and M <= 2 * I + 1]
    n_full = n_finite0 = n_end_out = 0
    for k, (I, M) in enumerate(shapes):
        kind = ("small", "full", "equal")[k % 3]
        fin, fmdl = band_rows(rng, I, kind), band_rows(rng, M, kind)
        full = full_dp_ref(fin, fmdl)
        for r in range(max(0, M - 1), 16):
            assert band_dp_ref(fin, fmdl, r) == full, (I, M, r)
            n_full += 1
        r0 = band_dp_ref(fin, fmdl, 0)
        assert r0 == band0_closed_form(fin, fmdl), (I, M)
        n_finite0 += r0 != DIS_ERR
        n_end_out += (r0 == DIS_ERR) and not guard_rejects(I, M)
        if I == M:
            assert r0 == int(np.trace(dist_matrix(fin, fmdl))) // (2 * I)
    assert n_full > 1000 and n_finite0 > 100 and n_end_out > 100


def test_dtw_band_oracle_equals_plain_reference_every_radius():
    """sro_dtw_band (through oracle_bind.port().dtw_batch) == band_dp_ref for every r in 0..15 on every (I, M) of the guard
    edges, 1x1, 1x2, 2x1, 119x119, 60x119 and 119x60, with small, full-range and all-equal features and the largest local
    distance"""
    po = ob.port()
    rng = np.random.default_rng(10)
    kinds = ("small", "full", "equal")
    for k, (I, M) in enumerate(guard_edge_shapes()):
        kind = kinds[k % 3]
        fin, fmdl = band_rows(rng, I, kind), band_rows(rng, M, kind)
        if (I, M) in ((119, 119), (60, 119), (119, 60)):
            fin, fmdl = np.tile(MAX_A, (I, 1)), np.tile(MAX_B, (M, 1))
        fi, fm = make_ftr([fin]), make_ftr([fmdl])
        for r in range(16):
            got = int(po.dtw_batch(fi, fm.view(np.uint8), 1, ob.FTR_DTYPE.itemsize, band_r=r)[0][0, 0])
            want = band_dp_ref(fin, fmdl, r)
            assert got == want, (I, M, kind, r, got, want)
    # the largest result any pair can have: every cell 65 536, 119 cells on the cheapest path
    res, D = band_dp_ref(np.tile(MAX_A, (119, 1)), np.tile(MAX_B, (119, 1)), 0, with_d=True)
    assert D == 119 * 65536 and res == D // 238


# ---- K3 on the GPU: both band kernels, every radius --------------------------------------------------------------
@pytest.mark.gpu
def test_dtw_band_kernels_equal_plain_reference_and_oracle_every_radius(handle):
    """sr_dtw_batch with SR_DTW_BAND for every r in 0..15 (the warp-scan kernel for 15 radii, the thread kernel for r = 10):
    score, best_idx and best_dis bit for bit against the oracle on every pair of four 119 x 119 cases, and against
    band_dp_ref on a sample of 448 pairs. The cases: small features; +-32 767 features, with the largest local distance on
    every cell of the 60- and 119-row sets (the largest path sums a result can have); all-equal features (D = 0, every min
    a tie); self-matches. r = 0 pairs whose end column lies outside the last row's band are dis_err. A wider band never
    raises a score that both radii reach."""
    po = ob.port()
    rng = np.random.default_rng(0x5EED)
    stride = ob.FTR_DTYPE.itemsize
    n_checked = 0
    for name, utt, tpl in band_cases():
        fin, bank = make_ftr(utt), make_ftr(tpl)
        B, T = len(fin), len(bank)
        I = fin["frm_num"].astype(np.int64)[:, None]
        M = bank["frm_num"].astype(np.int64)[None, :]
        walks = (I <= 2 * M) & (M <= 2 * I)
        handle.set_bank(bank.view(np.uint8).reshape(T, stride), T, stride)
        scores = []
        for r in range(16):
            score, bi, bd = handle.dtw(fin, flags=sr_b200.DTW_BAND, band_r=r)
            want, _ = po.dtw_batch(fin, bank.view(np.uint8), T, stride, band_r=r, nthreads=NTHREADS)
            assert np.array_equal(score, want), (name, r)
            key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
            k = key.min(axis=1)
            assert np.array_equal(bi, (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)), (name, r)
            assert np.array_equal(bd, (k >> np.uint64(32)).astype(np.uint32)), (name, r)
            # the plain reference on the corners (119x119, 60x119, 119x60, 1x1, 1x2, 2x1) and a few random pairs
            pairs = [(118, 118), (59, 118), (118, 59), (0, 0), (0, 1), (1, 0)]
            pairs += [tuple(p) for p in rng.integers(0, MAX_FRM, (1, 2))] + [tuple(rng.choice(np.argwhere(walks)))]
            for u, t in pairs:
                assert score[u, t] == band_dp_ref(utt[u], tpl[t], r), (name, r, u, t)
                n_checked += 1
            if r == 0:
                assert (score[walks & (M > I)] == DIS_ERR).all() and (score[walks & (M <= I)] != DIS_ERR).all()
            assert (score[~walks] == DIS_ERR).all() and (score[walks & (M <= r + 1)] != DIS_ERR).all()
            if name == "self":
                assert (np.diag(score) == 0).all()
            if name == "equal":
                assert (score[score != DIS_ERR] == 0).all()
            if name == "full":                   # max(I, M) cells of 65 536 on the cheapest path
                assert score[118, 118] == 119 * 65536 // 238 and score[118, 59] == 119 * 65536 // 179
                assert score[59, 59] == 60 * 65536 // 120 and score[59, 118] == (DIS_ERR if r == 0 else 119 * 65536 // 179)
            scores.append(score)
        S = np.stack(scores).astype(np.int64)
        reach = S != DIS_ERR
        assert (reach[1:] >= reach[:-1]).all(), name                     # reachable at r -> reachable at r + 1
        assert (np.where(reach[:-1], S[1:] <= S[:-1], True)).all(), name
        assert reach[0].sum() < reach[15].sum(), name
        if name in ("small", "full"):
            assert (reach[0] & (S[15] < S[0])).any(), name
    assert n_checked == 4 * 16 * 8


# ---- K5: the GEOM_B tables from their float64 formulas ------------------------------------------------------------
def _header_table(name):
    import re
    text = open(os.path.join(ob.ROOT, "stm32-speech-recognition_b200", "csrc", "sr_tables.h")).read()
    body = re.search(r"\b%s\[(\d+)\] = \{([^}]*)\}" % name, text)
    vals = [int(x) for x in body.group(2).replace("\n", "").split(",") if x.strip()]
    assert len(vals) == int(body.group(1))
    return np.array(vals, np.int64)


def test_geom_b_tables_follow_their_formulas():
    """sr_tab_b_hamm = round-half-away(10000 * hamming(200)) and symmetric; the 24 Mel centres strictly increase inside
    the 128 bins; every triangle weight lies in [0, 1000], each filter peaks at 1000 on its own centre (bin cen - 1: the
    tables are 0-based, the centres 1-based as in the Matlab source) and neighbouring triangles sum to 1000 between the
    first and the last centre"""
    hamm = _header_table("sr_tab_b_hamm")
    assert len(hamm) == 200 and np.array_equal(hamm, hamm[::-1])
    assert np.array_equal(hamm, np.floor(10000.0 * np.hamming(200) + 0.5).astype(np.int64))
    cen, odd, even = (_header_table("sr_tab_b_tri_" + n) for n in ("cen", "odd", "even"))
    assert len(cen) == 24 and len(odd) == 128 and len(even) == 128
    assert cen[0] >= 1 and (np.diff(cen) > 0).all() and cen[-1] < 128
    for tab in (odd, even):
        assert ((tab >= 0) & (tab <= 1000)).all()
    for h in range(24):
        assert (even if h % 2 == 0 else odd)[cen[h] - 1] == 1000, h
    lo, hi = cen[0] - 1, cen[-1] - 1
    assert ((odd + even)[lo:hi + 1] == 1000).all()


# ---- K5: the 256-point FFT against the exact DFT -------------------------------------------------------------------
def _pack(re, im):
    packed = (np.asarray(re, np.int64) & 0xFFFF) | ((np.asarray(im, np.int64) & 0xFFFF) << 16)
    return np.ascontiguousarray(packed, np.uint32)


def _unpack(packed):
    re = (packed & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.float64)
    im = (packed >> 16).astype(np.uint16).view(np.int16).astype(np.float64)
    return re, im


def _fft_inputs(N, rng, n=200):
    """random complex frames at amplitudes 2 000 .. 32 767 (half of them real), and for N = 256 real 200-sample frames
    zero-padded to 256 (the input the GEOM_B front end gives it)"""
    res, ims = [], []
    for amp in (2000, 8000, 16000, 32767):
        for real in (False, True):
            res.append(rng.integers(-amp, amp + 1, (n, N)))
            ims.append(np.zeros((n, N), np.int64) if real else rng.integers(-amp, amp + 1, (n, N)))
    if N == 256:
        re = np.zeros((2 * n, N), np.int64)
        re[:, :200] = rng.integers(-32767, 32768, (2 * n, 200))
        res.append(re)
        ims.append(np.zeros_like(re))
    return np.concatenate(res), np.concatenate(ims)


@pytest.mark.parametrize("N,bound", [(256, 8), (1024, 9)])
def test_generic_fft_is_within_a_few_lsb_of_the_exact_dft(N, bound):
    """cr4_fft_generic.c (the oracle's FFT for every size; at N = 1024 equal to the restated asm) against the float64
    DFT / N: at most `bound` LSB on either part of any bin (measured 6.8 at N = 256 and 8.2 at N = 1024 on these inputs; a
    wrong twiddle block, bit reversal or leg order gives errors in the hundreds)"""
    rng = np.random.default_rng(N)
    re, im = _fft_inputs(N, rng)
    got_re, got_im = _unpack(ob.port().fft_raw_n(_pack(re, im), N))
    want = dft_over_n(re, im)
    err = max(np.abs(got_re - want.real).max(), np.abs(got_im - want.imag).max())
    assert err <= bound, err


def _corner_frames(N):
    """frames of full-scale corner values c_k in {32767, -32768}^2 repeating with period 4 (c_{n mod 4}), as they are and
    with the sign flipped every 4 samples: all 256 choices of (c_0..c_3) each. Where the legs of a butterfly line up after
    their 45-degree twiddles, a part exceeds 32 767 and the s16 store wraps"""
    n = np.arange(N)
    corner = np.array([[32767, 32767], [32767, -32768], [-32768, 32767], [-32768, -32768]], np.int64)
    pick = np.array(list(np.ndindex(4, 4, 4, 4)))[:, n % 4]                   # [256, N]
    flip = np.where((n // 4) % 2 == 0, 1, -1)
    re = np.concatenate([corner[pick, 0], np.clip(corner[pick, 0] * flip, -32768, 32767)])
    im = np.concatenate([corner[pick, 1], np.clip(corner[pick, 1] * flip, -32768, 32767)])
    return re, im


def test_corner_frames_reach_the_s16_store_wrap():
    """the device FFT tests below use _corner_frames: on some of them the oracle's FFT is off the exact DFT / N by about
    2^16 (a store wrapped), on the others within the usual few LSB"""
    for N in (256, 1024):
        re, im = _corner_frames(N)
        got_re, got_im = _unpack(ob.port().fft_raw_n(_pack(re, im), N))
        want = dft_over_n(re, im)
        err = np.maximum(np.abs(got_re - want.real).max(axis=1), np.abs(got_im - want.imag).max(axis=1))
        wrapped = err > 30000
        assert 0 < wrapped.sum() < len(err) and (err[~wrapped] <= 9).all(), N


def _fft_device_inputs(N, rng):
    """arbitrary packed words, the all -32 768, all 0x7FFF and all 0 frames, the corner frames on which stores wrap, and
    the DFT test frames"""
    x = rng.integers(0, 2 ** 32, (64, N), dtype=np.uint64).astype(np.uint32)
    x[0], x[1], x[2], x[3] = 0x80008000, 0x7FFF7FFF, 0, 0x00007FFF
    x[4], x[5] = 0x80000000, 0x00008000
    re, im = _fft_inputs(N, rng, 16)
    cre, cim = _corner_frames(N)
    return np.ascontiguousarray(np.concatenate([x, _pack(re, im), _pack(cre, cim)]))


@pytest.mark.gpu
def test_device_fft_256_equals_oracle_bit_for_bit(handle):
    """fft_radix4<256> of the shared MFCC core (the GEOM_B FFT) run alone through sr_debug_fft_raw_n == the oracle's
    cr4_fft_generic.c at N = 256 on arbitrary packed input, the full-scale corners and frames whose stores wrap, bit for
    bit"""
    x = _fft_device_inputs(256, np.random.default_rng(2560))
    assert np.array_equal(handle.fft_raw_n(x, 256), ob.port().fft_raw_n(x, 256))


@pytest.mark.gpu
def test_device_fft_hook_at_1024_equals_the_drop_in_fft(handle):
    """the same hook at N = 1024 == sr_fft_raw_batch (fft_generic_kernel) == the oracle's generic FFT at N = 1024"""
    x = _fft_device_inputs(1024, np.random.default_rng(10240))
    got = handle.fft_raw_n(x, 1024)
    assert np.array_equal(got, handle.fft_raw(x))
    assert np.array_equal(got, ob.port().fft_raw_n(x, 1024))
