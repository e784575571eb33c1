"""Alignment along the banded DP (K3p, an extension the reference does not have; parity unpinned): the optimal warping
path of sr_dtw_path_batch and the DTW barycentre averaging of sr_average_bank.

CPU: the oracle's restatement (tests/oracle_ext/align.c) equals band_path_ref and average_ref, plain numpy / Python references
written here from the definitions in speech_recog.h that share no code with it; the paths' invariants and the averaging
properties. GPU: both calls equal the oracle bit for bit, the scores equal sr_dtw_batch's band scores, and the averaged
bank is one recognition accepts."""
import numpy as np
import pytest

import oracle_ext as ox
import oracle_bind as ob
import sr_b200
from test_extension_refs import (DIS_ERR, MAX_FRM, NTHREADS, _band_cases, _ftr, _guard_edge_shapes,
                                 _guard_rejects, _rows, dist_matrix)

RADII = (0, 1, 7, 10, 15, 16, 59, 118, 1000)
INT32_MAX = 2 ** 31 - 1
STRIDE = ob.FTR_DTYPE.itemsize
PATH_MAX = 237
ALIGN, AVG_UPDATE = 7, 8                 # tags of sr_timing_collect


# ---- references ---------------------------------------------------------------------------------------------------
def band_path_ref(fin, fmdl, r):
    """(score, path, D(I-1,M-1)): the whole I x M matrix in exact integers, +inf outside the band |j - floor(i*M/I)| <= r,
    then the trace-back from (I-1, M-1): the neighbour with the smallest D, ties to the diagonal, then (i, j-1), then
    (i-1, j). Rejected pairs: (DIS_ERR, [], None)"""
    I, M = len(fin), len(fmdl)
    if _guard_rejects(I, M) or I > MAX_FRM or M > MAX_FRM:
        return DIS_ERR, [], None
    d = dist_matrix(fin, fmdl).tolist()
    inf = float("inf")
    D = [[inf] * M for _ in range(I)]
    for i in range(I):
        c = i * M // I
        for j in range(max(0, c - r), min(M - 1, c + r) + 1):
            if i == 0 and j == 0:
                D[i][j] = d[0][0]
                continue
            best = min(D[i - 1][j - 1] if i and j else inf, D[i][j - 1] if j else inf, D[i - 1][j] if i else inf)
            if best != inf:
                D[i][j] = best + d[i][j]
    end = D[I - 1][M - 1]
    if end == inf:
        return DIS_ERR, [], None
    i, j, path = I - 1, M - 1, [(I - 1, M - 1)]
    while (i, j) != (0, 0):
        cand = [(D[i - 1][j - 1] if i and j else inf, 0), (D[i][j - 1] if j else inf, 1), (D[i - 1][j] if i else inf, 2)]
        k = min(cand)[1]                     # smallest D, then the lowest rank: diagonal, (i, j-1), (i-1, j)
        i, j = (i - 1, j - 1) if k == 0 else (i, j - 1) if k == 1 else (i - 1, j)
        path.append((i, j))
    return int(end) // (I + M), path[::-1], int(end)


def _slot_rows(slot):
    """(save_sign, frm_num, rows [frm_num, 12]) of a bank slot (rows only when frm_num <= 119)"""
    f = slot[:STRIDE].view(ob.FTR_DTYPE)[0]
    n = int(f["frm_num"])
    return int(f["save_sign"]), n, (f["mfcc_dat"][: n * 12].reshape(n, 12).astype(np.int64) if n <= MAX_FRM else None)


def average_ref(bank, slot_stride, K, r, iters, ranges=None):
    """sr_average_bank from its definition: (bank_out, score [G, K], anchor [G]). ranges: a list that receives, per group
    with members and iters >= 1, the (lo, hi) per template cell of the frames the last update averaged"""
    bank = np.asarray(bank, np.uint8).reshape(-1, slot_stride)
    G = bank.shape[0] // K
    out = np.full_like(bank, 0xFF)
    score, anchor = np.full((G, K), DIS_ERR, np.uint32), np.full(G, 0xFFFFFFFF, np.uint32)
    for g in range(G):
        rows = {}
        for k in range(K):
            sign, n, x = _slot_rows(bank[g * K + k])
            if sign == sr_b200.SAVE_MASK and 1 <= n <= MAX_FRM:
                rows[k] = x
        if not rows:
            continue
        S = {(l, k): band_path_ref(rows[l], rows[k], r)[0] for l in rows for k in rows if l != k}
        a = min(rows, key=lambda k: (sum(S[l, k] for l in rows if l != k), k))
        C = rows[a].copy()
        for _ in range(iters):
            tot, cnt = np.zeros_like(C), np.zeros(len(C), np.int64)
            lo, hi = np.full(C.shape, 1 << 20), np.full(C.shape, -(1 << 20))
            for l, x in rows.items():
                s, path, _ = band_path_ref(x, C, r)
                if s == DIS_ERR:
                    continue
                for i, j in path:
                    tot[j] += x[i]
                    cnt[j] += 1
                    lo[j], hi[j] = np.minimum(lo[j], x[i]), np.maximum(hi[j], x[i])
            if cnt.any():
                C = np.sign(tot) * (np.abs(tot) // cnt[:, None])         # C division truncates toward zero
                if ranges is not None:
                    ranges.append((g, lo, hi, C.copy()))
        M = len(C)
        out[g * K, :4] = np.frombuffer(np.array([sr_b200.SAVE_MASK, M], np.uint16).tobytes(), np.uint8)
        out[g * K, 4:4 + 24 * M] = np.frombuffer(C.astype(np.int16).tobytes(), np.uint8)
        for k, x in rows.items():
            score[g, k] = band_path_ref(x, C, r)[0]
        anchor[g] = a
    return out, score, anchor


# ---- inputs -------------------------------------------------------------------------------------------------------
def _slot(rows, stride, sign=sr_b200.SAVE_MASK, frm=None):
    s = np.full(stride, 0xFF, np.uint8)
    n = len(rows) if frm is None else frm
    s[:4] = np.frombuffer(np.array([sign, n], np.uint16).tobytes(), np.uint8)
    s[4:4 + rows.size * 2] = np.frombuffer(np.ascontiguousarray(rows, np.int16).tobytes(), np.uint8)
    return s


def _random_groups(rng, G, K, stride, fmin=3, fmax=24, plant=True):
    """G groups of K slots of random features (lengths fmin..fmax, some repetitions of one word plus noise); with plant,
    the invalid cases go into the first groups: an erased slot, frm_num 0, frm_num 120, an unsigned slot, a member the
    2:1 guard rejects against the others, and an all-empty group"""
    bank = np.full((G * K, stride), 0xFF, np.uint8)
    for g in range(G):
        n0 = int(rng.integers(fmin, fmax + 1))
        base = rng.integers(-3000, 3001, (n0, 12))
        for k in range(K):
            n = int(np.clip(n0 + rng.integers(-n0 // 3, n0 // 3 + 1), 1, MAX_FRM))
            idx = np.minimum((np.arange(n) * n0) // n, n0 - 1)
            rows = base[idx] + rng.integers(-400, 401, (n, 12))
            bank[g * K + k] = _slot(rows, stride)
    if plant and G >= 3:
        k_last = K - 1
        if K >= 2:
            bank[0 * K + k_last] = 0xFF                                           # erased
            bank[1 * K + k_last] = _slot(np.zeros((0, 12)), stride, frm=0)        # frm_num 0
        if K >= 3:
            bank[0 * K + 1] = _slot(rng.integers(-9, 9, (5, 12)), stride, frm=120)   # frm_num 120
            bank[1 * K + 1] = _slot(rng.integers(-3000, 3001, (10, 12)), stride, sign=0)   # unsigned
            n = _slot_rows(bank[2 * K])[1]
            bank[2 * K + 1] = _slot(rng.integers(-3000, 3001, (min(2 * n + 3, MAX_FRM), 12)), stride)   # guard rejects
        bank[(G - 1) * K:G * K] = 0xFF                                            # all empty
    return bank


# ---- CPU: the oracle against the references -------------------------------------------------------------------------
def _check_path_invariants(I, M, r, score, path, D, fin, fmdl):
    assert path[0] == (0, 0) and path[-1] == (I - 1, M - 1)
    steps = {(b[0] - a[0], b[1] - a[1]) for a, b in zip(path, path[1:])}
    assert steps <= {(1, 0), (0, 1), (1, 1)}, steps
    assert all(abs(j - i * M // I) <= r for i, j in path)
    assert max(I, M) <= len(path) <= I + M - 1
    d = dist_matrix(fin, fmdl)
    assert sum(int(d[i, j]) for i, j in path) == D
    assert score == D // (I + M)


def test_oracle_path_equals_plain_reference_on_guard_edges():
    """sro_dtw_path == band_path_ref (score, path bytes, length) on every (I, M) of the 2:1 guard's edges with small,
    +-32 767 and all-equal rows (every min a tie: the tie-break decides) at r in {0, 1, 7, 10, 15, 16, 59, 118, 1000};
    the paths start at (0, 0), end at (I-1, M-1), step by (1,0), (0,1) or (1,1), stay in the band, sum get_dis to
    D(I-1, M-1), and the score equals sro_dtw_band. band_path_ref runs once per distinct band (r and min(r, M - 1) select
    the same cells)"""
    ao, po = ox.align(), ob.port()
    rng = np.random.default_rng(0xA1)
    kinds = ("small", "full", "equal")
    n_paths = n_err = 0
    for k, (I, M) in enumerate(_guard_edge_shapes()):
        fin, fmdl = _rows(rng, I, kinds[k % 3]), _rows(rng, M, kinds[k % 3])
        fi, fm = _ftr([fin]), _ftr([fmdl])
        memo = {}
        for r in RADII:
            dis, path, plen = ao.dtw_path(fi, fm, r)
            eff = min(r, M - 1)
            if eff not in memo:
                memo[eff] = band_path_ref(fin, fmdl, eff)
            score, want_path, D = memo[eff]
            assert int(dis[0]) == score == int(po.dtw_batch(fi, fm.view(np.uint8), 1, STRIDE, band_r=r)[0][0, 0]), (I, M, r)
            L = int(plen[0])
            assert L == len(want_path), (I, M, r)
            assert (path[0, L:] == 0xFF).all()
            assert [tuple(x) for x in path[0, :L].tolist()] == want_path, (I, M, r)
            if score == DIS_ERR:
                n_err += 1
                continue
            _check_path_invariants(I, M, r, score, want_path, D, fin, fmdl)
            n_paths += 1
    assert n_paths > 1500 and n_err > 300


def test_oracle_self_match_path_is_the_diagonal():
    """a self-match's path is the diagonal at every radius, also for all-equal rows where every cell ties"""
    ao = ox.align()
    rng = np.random.default_rng(0xA2)
    for n in (1, 2, 7, 60, 119):
        for kind in ("small", "equal", "full"):
            x = _rows(rng, n, kind)
            f = _ftr([x])
            for r in RADII:
                dis, path, plen = ao.dtw_path(f, f, r)
                assert dis[0] == 0 and plen[0] == n
                assert (path[0, :n] == np.arange(n)[:, None]).all()
                s, p, _ = band_path_ref(x, x, r)
                assert s == 0 and p == [(i, i) for i in range(n)]


@pytest.mark.parametrize("K", (1, 2, 4, 7))
def test_oracle_average_equals_plain_reference(K):
    """sro_average_bank == average_ref (bank bytes, scores, anchors) on random groups with the invalid cases planted, for
    iters in {0, 1, 3} and r in {10, 118}"""
    ao = ox.align()
    rng = np.random.default_rng(0xA3 + K)
    stride = 2880
    bank = _random_groups(rng, 6, K, stride)
    for r in (10, 118):
        for iters in (0, 1, 3):
            got = ao.average_bank(bank, stride, K, r, iters)
            want = average_ref(bank, stride, K, r, iters)
            for a, b, what in zip(got, want, ("bank", "score", "anchor")):
                assert np.array_equal(a, b), (K, r, iters, what)
            assert (got[2][-1] == 0xFFFFFFFF) and (got[0][-K:] == 0xFF).all()
            if K > 1:
                assert (got[0].reshape(-1, K, stride)[:, 1:] == 0xFF).all()


def test_averaging_properties():
    """K = 1 returns the member; K identical members return that member; iters = 0 returns the anchor; every output
    coefficient lies within the range of the frames aligned to it"""
    ao = ox.align()
    rng = np.random.default_rng(0xA4)
    stride = 4096
    bank = _random_groups(rng, 8, 1, stride, plant=False)
    for iters in (0, 1, 3):
        out, score, anchor = ao.average_bank(bank, stride, 1, 16, iters)
        assert np.array_equal(out, bank) and (score == 0).all() and (anchor == 0).all()
    one = _random_groups(rng, 5, 1, stride, plant=False)
    same = np.repeat(one, 4, axis=0)
    out, score, anchor = ao.average_bank(same, stride, 4, 10, 3)
    assert np.array_equal(out[::4], one) and (out.reshape(5, 4, stride)[:, 1:] == 0xFF).all()
    assert (score == 0).all() and (anchor == 0).all()
    bank = _random_groups(rng, 10, 4, stride, plant=False)
    out, score, anchor = ao.average_bank(bank, stride, 4, 118, 0)
    for g in range(10):
        n = _slot_rows(bank[g * 4 + anchor[g]])[1]
        assert np.array_equal(out[g * 4, :4 + 24 * n], bank[g * 4 + anchor[g], :4 + 24 * n])
    ranges = []
    want = average_ref(bank, stride, 4, 15, 2, ranges=ranges)
    assert all(np.array_equal(a, b) for a, b in zip(ao.average_bank(bank, stride, 4, 15, 2), want))
    assert len(ranges) == 20
    for g, lo, hi, C in ranges:
        assert ((lo <= C) & (C <= hi)).all(), g


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _all_pairs(utt, tpl):
    """every (utterance u, template t) pair of a _band_cases case, u-major"""
    n = len(utt)
    fin, fm = _ftr(utt), _ftr(tpl)
    return np.repeat(fin, n), np.tile(fm, n)


@pytest.mark.gpu
def test_path_batch_equals_oracle_on_every_shape():
    """sr_dtw_path_batch == the oracle bit for bit (path bytes, lengths, scores) on all 119 x 119 shapes of the four
    _band_cases at r in {0, 1, 7, 10, 15, 16, 59, 118, 1000} and INT32_MAX (against r = 118); the scores equal
    sr_dtw_batch with SR_DTW_BAND for the same pairs; a NULL path gives the same scores; self-matches walk the diagonal"""
    ao = ox.align()
    h = sr_b200.Handle(0)
    for name, utt, tpl in _band_cases():
        a, b = _all_pairs(utt, tpl)
        bank = _ftr(tpl)
        h.set_bank(bank.view(np.uint8).reshape(len(tpl), STRIDE), len(tpl), STRIDE)
        for r in RADII + (INT32_MAX,):
            dis, path, plen = h.dtw_path(a, b, r)
            wdis, wpath, wlen = ao.dtw_path(a, b, min(r, 118), nthreads=NTHREADS)
            assert np.array_equal(dis, wdis), (name, r)
            assert np.array_equal(plen, wlen), (name, r)
            assert np.array_equal(path, wpath), (name, r)
            score, _, _ = h.dtw(_ftr(utt), flags=sr_b200.DTW_BAND, band_r=r, want_best=False)
            assert np.array_equal(dis.reshape(len(utt), len(tpl)), score), (name, r)
            assert np.array_equal(h.dtw_path(a, b, r, with_path=False)[0], dis), (name, r)
            if name == "self":
                n = np.arange(len(utt))
                diag = n * len(utt) + n
                assert (plen[diag] == n + 1).all() and (dis[diag] == 0).all()
    h.close()


@pytest.mark.gpu
def test_path_batch_argument_rules_and_timing():
    """a negative r fails; n = 0 launches nothing; one call is one launch, timed under tag 7"""
    h = sr_b200.Handle(0)
    h.timing_enable(16)
    rng = np.random.default_rng(0xA5)
    f = _ftr([_rows(rng, 20, "small"), _rows(rng, 33, "small")])
    for r in (-1, -1000):
        with pytest.raises(sr_b200.SrError):
            h.dtw_path(f, f, r)
    l0 = h.launch_count()
    h.dtw_path(f[:0], f[:0], 5)
    assert h.launch_count() == l0 and h.timing_collect() == []
    h.dtw_path(f, f[::-1].copy(), 5)
    assert h.launch_count() == l0 + 1 and [t for t, _ in h.timing_collect()] == [ALIGN]
    h.close()


@pytest.mark.gpu
def test_path_batch_does_not_depend_on_batch_position():
    """slices cut at and around multiples of SMs x warps per CTA (the persistent grid's stride) and of the CTA's 8 warps:
    every pair equals the oracle wherever it sits in the batch"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ao = ox.align()
    rng = np.random.default_rng(0xA6)
    n = 2 * sms * 2 * 8 + 50
    lens_a, lens_b = rng.integers(1, 120, n), rng.integers(1, 120, n)
    lens_b = np.clip(lens_b, (lens_a + 1) // 2, 2 * lens_a).clip(1, 119)
    a = _ftr([_rows(rng, int(x), "small") for x in lens_a])
    b = _ftr([_rows(rng, int(x), "small") for x in lens_b])
    h = sr_b200.Handle(0)
    for r in (7, 118):
        wdis, wpath, wlen = ao.dtw_path(a, b, r, nthreads=NTHREADS)
        cuts = sorted({0, n} | {c + e for c in (8, sms * 16, 2 * sms * 16) for e in (-1, 0, 1)})
        for lo, hi in zip(cuts, cuts[1:]):
            dis, path, plen = h.dtw_path(a[lo:hi], b[lo:hi], r)
            assert np.array_equal(dis, wdis[lo:hi]) and np.array_equal(plen, wlen[lo:hi]), (r, lo, hi)
            assert np.array_equal(path, wpath[lo:hi]), (r, lo, hi)
    h.close()


def _check_average(h, bank, stride, K, r, iters):
    """sr_average_bank against the oracle; scores against sr_dtw_batch(SR_DTW_BAND | SR_DTW_CHECK_SIGN) of every member
    against the output bank, which sr_set_bank accepts; 2 * iters + 3 launches, tags 7 and 8"""
    h.timing_collect()
    l0 = h.launch_count()
    got = h.average_bank(bank, stride, K, r, iters)
    launches, tags = h.launch_count() - l0, [t for t, _ in h.timing_collect()]
    want = ox.align().average_bank(bank, stride, K, r, iters, nthreads=NTHREADS)
    for a, b, what in zip(got, want, ("bank", "score", "anchor")):
        assert np.array_equal(a, b), (K, r, iters, what)
    out, score, anchor = got
    assert launches == 2 * iters + 3, (launches, iters)
    assert tags == [ALIGN] + [ALIGN, AVG_UPDATE] * iters + [ALIGN]
    G = len(anchor)
    h.set_bank(out, G * K, stride)
    hdr = bank.reshape(G * K, stride)[:, :4].copy().view(np.uint16)
    member = (hdr[:, 0] == sr_b200.SAVE_MASK) & (hdr[:, 1] >= 1) & (hdr[:, 1] <= MAX_FRM)
    inputs = np.ascontiguousarray(bank.reshape(G * K, stride)[member, :STRIDE]).view(ob.FTR_DTYPE).reshape(-1)
    s, _, _ = h.dtw(inputs, flags=sr_b200.DTW_BAND | sr_b200.DTW_CHECK_SIGN, band_r=r, want_best=False)
    slots = np.flatnonzero(member)
    assert np.array_equal(s[np.arange(len(slots)), (slots // K) * K], score.reshape(-1)[slots])
    assert (score.reshape(-1)[~member] == DIS_ERR).all()
    return got


@pytest.mark.gpu
def test_average_bank_enrolled_groups_equal_oracle():
    """300 groups of 4 slots from sr_enrol_batch on synthetic PCM (failed enrolments leave erased slots)"""
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    h.set_transport(0)
    bank, st = h.enrol(sr_b200.synth_pcm_host(1200, 8000, 0xAB0000), 2400)
    assert (st == 0).sum() > 1000
    for r, iters in ((10, 0), (10, 1), (118, 3), (16, 2)):
        out, score, anchor = _check_average(h, bank, 4096, 4, r, iters)
        assert (anchor != 0xFFFFFFFF).sum() > 250
    h.close()


@pytest.mark.gpu
def test_average_bank_random_groups_with_invalid_slots_equal_oracle():
    """70 groups of random features with an erased slot, frm_num 0, frm_num 120, an unsigned slot, a member the 2:1
    guard rejects and an all-empty group planted, K in {1, 4, 7, 32}"""
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    for K in (4, 7, 32):
        bank = _random_groups(np.random.default_rng(0xA7 + K), 70, K, 4096, fmin=5, fmax=119)
        for r, iters in ((10, 0), (118, 1), (15, 3)):
            _check_average(h, bank, 4096, K, r, iters)
    bank = _random_groups(np.random.default_rng(0xA8), 70, 1, 2880, plant=False)
    got = h.average_bank(bank, 2880, 1, 16, 2)
    assert np.array_equal(got[0], bank)
    assert all(np.array_equal(a, b) for a, b in zip(got, ox.align().average_bank(bank, 2880, 1, 16, 2)))
    with pytest.raises(sr_b200.SrError):
        h.average_bank(bank, 2880, 1, -1, 1)
    h.close()
