"""The template matchers at the inputs where a wrong kernel still passes random features: unique minima, the any-rate
slides of the register band, first-wins ties across a reordered bank, the anchor and arithmetic edges of the averaging,
and the path call's empty and oversized inputs. Each case is checked bit for bit against the oracles of tests/oracle_ext
and the plain references of refs.py; a CPU test proves that each plant reaches its case (the minimum is unique, the slide
reaches s, the tie really ties) before the GPU relies on it.
DESIGN.md lists the mutants of K2, K3, K3p, K6 and the shared core, and the test that catches each."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import make_ftr, make_slot
from refs import (DIS_ERR, MAX_FRM, NTHREADS, STRIDE, average_ref, band_dp_ref, band_matrix, band_path_ref, rate_ref,
                  slot_rows, want_best)

BAND, ANY = sr_b200.DTW_BAND, sr_b200.DTW_ANY_RATE
ALIGN, AVG_UPDATE = 7, 8                     # tags of sr_timing_collect
RADII = (0, 1, 9, 10, 11, 15, 16, 118)      # both edges of each band kernel: warp-scan (<= 15), thread (10), whole row
R = 10                                       # the thread form's radius; its band holds W = 21 cells
W = 2 * R + 1


# ---- plant checks -------------------------------------------------------------------------------------------------
def ties(D):
    """reachable cells whose smallest predecessor is not unique"""
    inf, n = float("inf"), 0
    for i in range(len(D)):
        for j in range(len(D[0])):
            if D[i][j] == inf or (i == 0 and j == 0):
                continue
            p = sorted([D[i - 1][j - 1] if i and j else inf, D[i][j - 1] if j else inf, D[i - 1][j] if i else inf])
            n += p[0] == p[1]
    return n


# ---- unique-minimum features ----------------------------------------------------------------------------------------
UNIQUE_LENS = (1, 2, 3, 7, 12, 30, 59, 60, 61, 118, 119)


def _wide_rows(rng, n):
    """rows of +-9 000: every squared distance stays below 2^32 (no wrap), so local distances spread over 0 .. 62 000"""
    return rng.integers(-9000, 9001, (n, 12)).astype(np.int16)


def unique_case():
    rng = np.random.default_rng(0xE1)
    utt = [_wide_rows(rng, n) for n in UNIQUE_LENS]
    tpl = [_wide_rows(rng, n) for n in UNIQUE_LENS[::-1]]
    return utt, tpl


def test_unique_minimum_features_rarely_tie():
    """on the pairs of the unique-minimum case (ratios up to 119:1 both ways) at every radius, all but at most 1 in 10 000
    reachable cells have a smallest predecessor strictly below the other two, so a wrong predecessor, mask edge or clamp
    changes D; most pairs reach their end cell at every radius"""
    utt, tpl = unique_case()
    n_end = n_tie = n_cell = 0
    for x in utt:
        for y in tpl:
            for r in RADII:
                D = band_matrix(x, y, r)
                n_tie += ties(D)
                n_cell += sum(v != float("inf") for row in D for v in row)
                n_end += D[-1][-1] != float("inf")
    assert n_cell > 500000 and n_tie * 10000 < n_cell, (n_tie, n_cell)
    assert n_end > 0.6 * len(utt) * len(tpl) * len(RADII)


@pytest.mark.gpu
def test_unique_minimum_features_every_band_kernel():
    """sr_dtw_batch(BAND) and (BAND | ANY_RATE) at r = 0, 1, 9, 10, 11, 15, 16, 118 on the unique-minimum case: scores and
    argmin against the port's band DP and the any-rate oracle, and every pair against band_dp_ref / rate_ref"""
    utt, tpl = unique_case()
    fin, bank = make_ftr(utt), sr_b200.make_bank(make_ftr(tpl), STRIDE)
    po, ro = ob.port(), ox.rate_oracle()
    h = sr_b200.Handle(0)
    h.set_bank(bank, len(tpl), STRIDE)
    try:
        for r in RADII:
            for flags in (BAND, BAND | ANY):
                score, bi, bd = h.dtw(fin, flags=flags, band_r=r)
                if flags & ANY:
                    want = ro.dtw_batch(fin, bank, len(tpl), STRIDE, band_r=r, nthreads=NTHREADS)
                else:
                    want, _ = po.dtw_batch(fin, bank, len(tpl), STRIDE, band_r=r, nthreads=NTHREADS)
                assert np.array_equal(score, want), (r, flags, np.argwhere(score != want)[:4].tolist())
                wi, wd = want_best(want)
                assert np.array_equal(bi, wi) and np.array_equal(bd, wd), (r, flags)
                for u, x in enumerate(utt):
                    for t, y in enumerate(tpl):
                        if flags & ANY:
                            d = rate_ref(x, y, r)
                            ref = DIS_ERR if d is None else d // (len(x) + len(y))
                        else:
                            ref = band_dp_ref(x, y, r)
                        assert score[u, t] == ref, (r, flags, len(x), len(y))
    finally:
        h.close()


# ---- any-rate slides of the thread form (r = 10) --------------------------------------------------------------------
def thread_rows(I, M):
    """the thread form's walk over the rows of an (I, M) pair: (i, slide s = c_i - c_{i-1}, catch-up division taken)"""
    c = cprev = err = 0
    out = []
    for i in range(I):
        out.append((i, c - cprev, False))
        cprev = c
        err += M
        for _ in range(2):
            if err >= I:
                err -= I
                c += 1
        if err >= I:
            out[-1] = (i, out[-1][1], True)
            c += err // I
            err %= I
    return out


def slide_shapes():
    """every I in 1..59 against M = 2I + 1, 3I, 22I and 119 (capped at 119), and M = sI for every slide s = 3 .. 22 at
    I = 2 .. 5: slides of 3 .. 59 columns"""
    shapes = {(I, min(m, MAX_FRM)) for I in range(1, 60) for m in (2 * I + 1, 3 * I, 22 * I, MAX_FRM)}
    return sorted(shapes | {(I, s * I) for I in range(2, 6) for s in range(3, 23) if s * I <= MAX_FRM})


def slide_case():
    """one (utterance, template) pair per slide shape. In the first row i >= 1 whose slide s is 3 .. 21 the left band
    edge's diagonal source, old index s - 1 = column c_i - R - 1 of row i - 1, is planted cheap: utterance rows i - 1 and
    i equal template columns c_i - R - 1 and c_i - R. Returns (pairs, the planted cell (i, c_i - R) per pair or None)"""
    rng = np.random.default_rng(0xE2)
    pairs, plants = [], []
    for I, M in slide_shapes():
        x, y = _wide_rows(rng, I), _wide_rows(rng, M)
        plant = None
        for i, s, _ in thread_rows(I, M):
            c = i * M // I
            if i >= 1 and 3 <= s <= W and c - R - 1 >= 0:
                x[i - 1], x[i] = y[c - R - 1], y[c - R]
                plant = (i, c - R)
                break
        pairs.append((x, y))
        plants.append(plant)
    return pairs, plants


def test_slide_case_reaches_every_slide_and_catch_up():
    """the thread form's incremental centre is floor(i*M/I) on every row; the slide shapes reach every slide 3 .. 21 and
    slides past W = 21, and the catch-up division runs for every I in 1..59; in each planted pair the left edge's diagonal
    from old index s - 1 is reachable and the unique minimum of its cell (the cell's left neighbour lies outside the band)"""
    slides, catch = set(), set()
    for I, M in slide_shapes():
        for i, s, cu in thread_rows(I, M):
            assert s == i * M // I - (i - 1) * M // I if i else s == 0
            slides.add(s)
            if cu:
                catch.add(I)
    assert set(range(3, W + 1)) <= slides and max(slides) > W + 30
    assert catch == set(range(1, 60))
    pairs, plants = slide_case()
    n = 0
    for (x, y), p in zip(pairs, plants):
        if p is None:
            continue
        i, j = p
        D = band_matrix(x, y, R)
        assert D[i - 1][j - 1] < float("inf") and D[i - 1][j - 1] < D[i - 1][j], (len(x), len(y), i)
        assert j - 1 < i * len(y) // len(x) - R                     # the left neighbour (i, j - 1) is outside the band
        n += 1
    assert n >= 50


@pytest.mark.gpu
def test_thread_form_slides_equal_oracle_and_plain_reference():
    """sr_dtw_batch(BAND | ANY_RATE, r = 10) on every pair of the slide case (and the cross pairs of the batch) against the
    any-rate oracle, and each planted pair against rate_ref; plain BAND at r = 10 rejects the pairs past 2:1"""
    pairs, plants = slide_case()
    utt = [p[0] for p in pairs]
    tpl = [p[1] for p in pairs]
    fin, bank = make_ftr(utt), sr_b200.make_bank(make_ftr(tpl), STRIDE)
    T = len(tpl)
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, STRIDE)
    try:
        score, bi, bd = h.dtw(fin, flags=BAND | ANY, band_r=R)
        want = ox.rate_oracle().dtw_batch(fin, bank, T, STRIDE, band_r=R, nthreads=NTHREADS)
        assert np.array_equal(score, want), np.argwhere(score != want)[:4].tolist()
        wi, wd = want_best(want)
        assert np.array_equal(bi, wi) and np.array_equal(bd, wd)
        for k, (x, y) in enumerate(pairs):
            d = rate_ref(x, y, R)
            assert score[k, k] == (DIS_ERR if d is None else d // (len(x) + len(y))), (len(x), len(y))
        assert (np.diag(score) != DIS_ERR).sum() > 50
        plain, _, _ = h.dtw(fin, flags=BAND, band_r=R)
        assert (np.diag(plain) == DIS_ERR).all()
    finally:
        h.close()


# ---- first wins across a reordered bank -----------------------------------------------------------------------------
def tie_bank(T):
    """all-equal rows (every local distance 0, every score 0): slot 0 holds the longest template (119 frames) and slot
    T - 1 a duplicate of it, the other slots 60..118 frames, so the bank order (ascending frm_num, stable) visits every
    other slot before slot 0 and its duplicate last: at T = 33 slot 0 is the last of the first full tile and its
    duplicate the remainder tile"""
    row = np.array([7, -3, 11, 0, -25, 4, 9, -1, 2, 3, -8, 6], np.int16)
    lens = [MAX_FRM] + [60 + (k * 37) % 59 for k in range(1, T - 1)] + [MAX_FRM]
    return sr_b200.make_bank(make_ftr([np.tile(row, (n, 1)) for n in lens]), STRIDE), lens, row


def tie_inputs(row):
    return make_ftr([np.tile(row, (n, 1)) for n in (60, 80, 100, 119)])


def test_tie_bank_ties_everywhere_and_is_visited_out_of_order():
    """every pair of the tie banks scores 0 in the greedy and band oracles, and the walk order sr_set_bank derives from
    the headers puts slot 0 after a higher slot in a later tile"""
    po = ob.port()
    for T in (33, 70, 200):
        bank, lens, row = tie_bank(T)
        fin = tie_inputs(row)
        for r in (-1, 5, 10, 16):
            want, _ = po.dtw_batch(fin, bank, T, STRIDE, band_r=r)
            assert (want == 0).all(), (T, r)
        order = sorted(range(T), key=lambda k: lens[k])
        assert order.index(0) == T - 2 and order.index(T - 1) == T - 1


@pytest.mark.gpu
@pytest.mark.parametrize("T", (33, 70, 200))
def test_first_wins_across_reordered_bank(T):
    """on the tie banks every kernel reports best_idx 0 and best_dis 0: the static and dynamic greedy walk, the warp-scan
    (r = 5), thread (r = 10) and whole-row (r = 16) band kernels, with and without ANY_RATE, from a host bank and from a
    device bank set twice at the same address (the second call keeps the cached order)"""
    import torch
    bank, lens, row = tie_bank(T)
    fin = tie_inputs(row)
    dev = torch.from_numpy(bank.reshape(-1)).cuda()
    h = sr_b200.Handle(0)
    try:
        for where in ("host", "dev", "dev again"):
            if where == "host":
                h.set_bank(bank, T, STRIDE)
            else:
                torch.cuda.synchronize()
                h.set_bank_dev(dev.data_ptr(), T, STRIDE)
            runs = [(0, 0, v) for v in (0, 1)] + [(f, r, None) for r in (5, 10, 16) for f in (BAND, BAND | ANY)]
            for flags, r, variant in runs:
                if variant is not None:
                    h.set_dtw_variant(variant)
                score, bi, bd = h.dtw(fin, flags=flags, band_r=r)
                assert (score == 0).all(), (where, flags, r, variant)
                assert (bi == 0).all() and (bd == 0).all(), (where, flags, r, variant, bi.tolist())
        h.set_dtw_variant(-1)
    finally:
        h.close()


# ---- a failed utterance against a 0-frame template --------------------------------------------------------------------
FAILED_U, ZERO_SLOT = 3, 2


def failed_case():
    """five synthetic utterances, utterance 3 silent (constant PCM: the VAD finds no segment, so it has 0 frames), and a
    bank of six templates of 20..40 frames whose slot 2 is signed with frm_num 0. The 2:1 guard admits a 0:0 pair, so
    only the status gate keeps the greedy walk off the failed utterance's pair with slot 2"""
    rng = np.random.default_rng(0xE7)
    pcm = sr_b200.synth_pcm_host(5, 8000, 0xFA11ED00)
    pcm[FAILED_U] = 2048
    bank = sr_b200.make_bank(make_ftr([rng.integers(-3000, 3001, (int(n), 12)) for n in rng.integers(20, 41, 6)]), 4096)
    bank[ZERO_SLOT] = make_slot(np.zeros((0, 12)), 4096, frm=0)
    return pcm, bank


def test_failed_case_plants():
    """the reference fails the silent utterance and scores its row SR_DIS_ERR, and its greedy dtw walks a 0-frame input
    against slot 2 to a score"""
    pcm, bank = failed_case()
    ora = ob.best_oracle()
    ref = ora.recognise_batch(pcm, 2400, bank, len(bank), 4096)
    assert ref["status"][FAILED_U] != 0 and (np.delete(ref["status"], FAILED_U) == 0).all()
    assert (ref["score"][FAILED_U] == DIS_ERR).all()
    empty = make_ftr([np.zeros((0, 12), np.int16)])
    assert ora.dtw_batch(empty, bank, len(bank), 4096)[0][0, ZERO_SLOT] != DIS_ERR


@pytest.mark.gpu
def test_failed_utterance_against_a_zero_frame_template():
    """recognition with the static and the dynamic greedy kernel equals the reference's spch_recg on the failed case, so
    the failed utterance's pair with the 0-frame slot is SR_DIS_ERR and not a walk; the band matcher at r = 5, 10 and 16
    scores the failed row SR_DIS_ERR too"""
    pcm, bank = failed_case()
    T = len(bank)
    ref = ob.best_oracle().recognise_batch(pcm, 2400, bank, T, 4096)
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    try:
        for variant in (0, 1):
            h.set_dtw_variant(variant)
            out = h.recognise(pcm, 2400)
            for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
                assert np.array_equal(out[k].reshape(-1), ref[k].reshape(-1)), (variant, k)
            assert (out["score"][FAILED_U] == DIS_ERR).all(), variant
        h.set_dtw_variant(-1)
        for r in (5, 10, 16):
            h.set_match(BAND, r)
            out = h.recognise(pcm, 2400, want=("score", "status"))
            assert out["status"][FAILED_U] != 0 and (out["score"][FAILED_U] == DIS_ERR).all(), r
    finally:
        h.close()


# ---- averaging: anchors, arithmetic, passes -------------------------------------------------------------------------
AVG_R = 3                                    # a radius below 118: S(l -> k) and S(k -> l) differ


def _group_slots(members, K, stride=STRIDE):
    """one group of K slots: members {k: rows}, the other slots erased"""
    g = np.full((K, stride), 0xFF, np.uint8)
    for k, rows in members.items():
        g[k] = make_slot(rows, stride)
    return g


def anchor_bank():
    """G groups of K = 32: (0) identical members in every slot, (1) identical members with slot 0 erased, (2..33) a single
    member at k = 0 .. 31, (34) six members of 1, 3, 7, 15, 31 and 63 frames at k = 26..31 (every pair past 2:1: each
    S(l -> k) is SR_DIS_ERR and every sum saturated), (35) the same six at k = 1, 5, 9, 20, 30, 31"""
    rng = np.random.default_rng(0xE3)
    same = rng.integers(-3000, 3001, (17, 12))
    groups = [_group_slots({k: same for k in range(32)}, 32), _group_slots({k: same for k in range(1, 32)}, 32)]
    for k in range(32):
        groups.append(_group_slots({k: rng.integers(-3000, 3001, (int(rng.integers(1, 120)), 12))}, 32))
    chain = [rng.integers(-3000, 3001, (n, 12)) for n in (1, 3, 7, 15, 31, 63)]
    groups.append(_group_slots(dict(zip(range(26, 32), chain)), 32))
    groups.append(_group_slots(dict(zip((1, 5, 9, 20, 30, 31), chain)), 32))
    return np.concatenate(groups)


ANCHORS = [0, 1] + list(range(32)) + [26, 1]


def test_anchor_bank_plants():
    """average_ref's anchors are the planted ones; in the identical groups every S is 0, in the chain groups every S of
    two members is SR_DIS_ERR (sums of 5 * (2^32 - 1)), so the anchor is the lowest member and not k = 0"""
    bank = anchor_bank()
    out, score, anchor = average_ref(bank, STRIDE, 32, AVG_R, 1)
    assert anchor.tolist() == ANCHORS
    same = slot_rows(bank[0])[2]
    assert band_path_ref(same, same, AVG_R)[0] == 0
    chain = [slot_rows(bank[34 * 32 + k])[2] for k in range(26, 32)]
    for a in chain:
        for b in chain:
            if a is not b:
                assert band_path_ref(a, b, AVG_R)[0] == DIS_ERR
    assert (score[34, 27:] == DIS_ERR).all() and score[34, 26] == 0      # only the anchor aligns to C, which stays


def arithmetic_bank():
    """groups of K = 4 at the s16 extremes: (0) +-32 767 and -32 768 rows, (1) members whose column sums are negative and
    not multiples of their count, (2) a member twice as long as the others whose first rows all align to template column 0
    (the most frames one path puts into one column: I - M + 1)"""
    rng = np.random.default_rng(0xE4)
    ext = [np.where(rng.random((20, 12)) < 0.5, 32767, -32768) for _ in range(4)]
    ext[1][:, :6] = -32767
    neg = [rng.integers(-3000, 1, (25, 12)) for _ in range(4)]
    base = rng.integers(-3000, 3001, (30, 12))
    long = np.concatenate([np.tile(base[0], (31, 1)), base[1:]])        # 60 rows: rows 0..30 all equal column 0's
    vert = {0: base, 1: base + 1, 2: long, 3: base - 1}
    return np.concatenate([_group_slots(dict(enumerate(ext)), 4), _group_slots(dict(enumerate(neg)), 4),
                           _group_slots(vert, 4)])


def _sums(bank, K, r, g):
    """(sum, count) per template cell of group g's first update, from band_path_ref paths against its anchor"""
    _, _, anchor = average_ref(bank, STRIDE, K, r, 0)
    C0 = slot_rows(bank[g * K + anchor[g]])[2]
    tot, cnt = np.zeros_like(C0), np.zeros(len(C0), np.int64)
    for k in range(K):
        _, n, x = slot_rows(bank[g * K + k])
        if x is None or n == 0:
            continue
        s, path, _ = band_path_ref(x, C0, r)
        for i, j in path:
            tot[j] += x[i]
            cnt[j] += 1
    return tot, cnt


def test_arithmetic_bank_plants():
    """group 1 has negative column sums whose truncated and floored quotients differ; in group 2 column 0 receives
    I - M + 1 = 31 frames of the long member's path; group 0 sums rows of -32 768 and 32 767"""
    bank = arithmetic_bank()
    for r in (AVG_R, 118):
        tot, cnt = _sums(bank, 4, r, 1)
        q = tot / cnt[:, None]
        assert ((tot < 0) & (np.trunc(q) != np.floor(q))).any(), r
    _, _, anchor = average_ref(bank, STRIDE, 4, 118, 0)
    C0 = slot_rows(bank[2 * 4 + anchor[2]])[2]
    _, path, _ = band_path_ref(slot_rows(bank[2 * 4 + 2])[2], C0, 118)
    assert len(C0) == 30 and sum(1 for _, j in path if j == 0) == 60 - 30 + 1
    assert (slot_rows(bank[0])[2] == -32768).any() and (slot_rows(bank[0])[2] == 32767).any()


def _average_and_count(h, bank, K, r, iters):
    h.timing_collect()
    l0 = h.launch_count()
    got = h.average_bank(bank, STRIDE, K, r, iters)
    return got, h.launch_count() - l0, [t for t, _ in h.timing_collect()]


@pytest.mark.gpu
def test_average_bank_anchor_and_arithmetic_edges():
    """sr_average_bank on the anchor and arithmetic banks at r = 3 and 118, iters 0 .. 2, bit for bit against the oracle and
    average_ref: the planted anchors, C unchanged where only the anchor aligns, and 2 * iters + 3 launches"""
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    ao = ox.align()
    try:
        for bank, K in ((anchor_bank(), 32), (arithmetic_bank(), 4)):
            for r in (AVG_R, 118):
                for iters in (0, 1, 2):
                    got, launches, tags = _average_and_count(h, bank, K, r, iters)
                    want = ao.average_bank(bank, STRIDE, K, r, iters, nthreads=NTHREADS)
                    ref = average_ref(bank, STRIDE, K, r, iters)
                    for a, b, c, what in zip(got, want, ref, ("bank", "score", "anchor")):
                        assert np.array_equal(a, b) and np.array_equal(a, c), (K, r, iters, what)
                    assert launches == 2 * iters + 3 and tags == [ALIGN] + [ALIGN, AVG_UPDATE] * iters + [ALIGN]
                    if K == 32:
                        assert got[2].tolist() == ANCHORS
                        assert np.array_equal(got[0][34 * 32], bank[34 * 32 + 26])      # C = the anchor, unchanged
    finally:
        h.close()


@pytest.mark.gpu
def test_average_bank_pass_counts():
    """K = 1 has no anchor scores: 2 * iters + 2 launches; a bank with no member launches only the packing (untimed) and
    returns erased slots and no anchor"""
    rng = np.random.default_rng(0xE5)
    one = np.concatenate([_group_slots({0: rng.integers(-3000, 3001, (n, 12))}, 1) for n in (1, 2, 50, 119)])
    empty = np.full((3 * 4, STRIDE), 0xFF, np.uint8)
    empty[1] = make_slot(np.zeros((0, 12)), STRIDE, frm=0)
    empty[2] = make_slot(rng.integers(-9, 9, (5, 12)), STRIDE, frm=120)
    empty[3] = make_slot(rng.integers(-3000, 3001, (10, 12)), STRIDE, sign=0)
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    try:
        for iters in (0, 1, 3):
            got, launches, tags = _average_and_count(h, one, 1, AVG_R, iters)
            assert np.array_equal(got[0], one) and (got[1] == 0).all() and (got[2] == 0).all()
            assert launches == 2 * iters + 2 and tags == [ALIGN, AVG_UPDATE] * iters + [ALIGN], (iters, launches, tags)
            got, launches, tags = _average_and_count(h, empty, 4, AVG_R, iters)
            assert (got[0] == 0xFF).all() and (got[1] == DIS_ERR).all() and (got[2] == 0xFFFFFFFF).all()
            assert launches == 1 and tags == [], (iters, launches, tags)
    finally:
        h.close()


# ---- the path call: empty and oversized inputs, path NULL --------------------------------------------------------------
def _path_inputs():
    """pairs 0 and 1 have 0 frames on one side; in pair 2 the input and in pair 4 the template says 120 frames (past
    vv_frm_max) against a partner the 2:1 guard admits (119 and 80 frames), so only the frame count rejects them"""
    rng = np.random.default_rng(0xE6)
    a = make_ftr([rng.integers(-3000, 3001, (n, 12)) for n in (0, 5, 119, 60, 80)])
    b = make_ftr([rng.integers(-3000, 3001, (n, 12)) for n in (5, 0, 119, 59, 80)])
    a["frm_num"][2] = 120
    b["frm_num"][4] = 120
    return a, b


def test_path_inputs_are_rejected_by_the_frame_count_alone():
    """the 120-frame pairs are within 2:1 and score SR_DIS_ERR in the oracle; the same rows with their true counts (119
    and 80) score"""
    a, b = _path_inputs()
    ao = ox.align()
    for k in (2, 4):
        assert max(a["frm_num"][k], b["frm_num"][k]) <= 2 * min(a["frm_num"][k], b["frm_num"][k])
    assert (ao.dtw_path(a, b, 118)[0][[2, 4]] == DIS_ERR).all()
    a2, b2 = a.copy(), b.copy()
    a2["frm_num"][2], b2["frm_num"][4] = 119, 80
    assert (ao.dtw_path(a2, b2, 118)[0][[2, 4]] != DIS_ERR).all()


@pytest.mark.gpu
def test_path_call_empty_oversized_and_null_path():
    """pairs with 0 or 120 frames on either side are SR_DIS_ERR with L = 0 and an all-0xFF path; the others equal the
    oracle; with path NULL and path_len given the lengths are still written and equal the oracle's"""
    a, b = _path_inputs()
    n = len(a)
    h = sr_b200.Handle(0)
    try:
        for r in (0, 10, 118):
            dis, path, plen = h.dtw_path(a, b, r)
            wdis, wpath, wlen = ox.align().dtw_path(a, b, r)
            assert np.array_equal(dis, wdis) and np.array_equal(plen, wlen) and np.array_equal(path, wpath), r
            bad = [0, 1, 2, 4]
            assert (dis[bad] == DIS_ERR).all() and (plen[bad] == 0).all() and (path[bad] == 0xFF).all()
            assert dis[3] != DIS_ERR and plen[3] >= 60
            dis2, len2 = np.zeros(n, np.uint32), np.full(n, 0xA5A5A5A5, np.uint32)
            aa, bb = np.ascontiguousarray(a), np.ascontiguousarray(b)
            rc = sr_b200.lib().sr_dtw_path_batch(h._h, aa.ctypes.data_as(C.c_void_p), bb.ctypes.data_as(C.c_void_p), n,
                                                 int(r), None, len2.ctypes.data_as(C.c_void_p),
                                                 dis2.ctypes.data_as(C.c_void_p))
            assert rc == 0 and np.array_equal(dis2, dis) and np.array_equal(len2, plen), r
    finally:
        h.close()
