"""The symmetric slope-constrained DP of Sakoe & Chiba (SR_DTW_SYM_P1, an extension the reference does not have; parity
unpinned) in sr_dtw_batch and as the matcher of every recognition call (sr_set_match).

CPU: the C oracle (tests/oracle_ext/sym.c) equals a plain Python cell-level reference, and a brute-force enumeration of every
P = 1 path (each complete path weighs I + M, the cheapest one is g); a planted band-edge case and the 65 536 headroom.
GPU: sr_dtw_batch under SR_DTW_SYM_P1 equals the oracle bit for bit at every radius, bank width and shape; the setter
rules; every recognition path under the matcher equals the oracle composition (front end, the C oracle's scores, the strict
'<' first-wins argmin, cmd = idx / 4); the matcher switched between pushes; tag 14 where tag 6 is under the band matcher;
threads; real speech, reported. sr_recognise_batch_dev_allgather is run on a one-rank communicator by test_decision_paths.py.
Every GPU test makes its own handles, so the session handle never carries a matcher."""
import itertools
import os
import threading

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import bank_planted, inputs, make_ftr, real_speech_pairs, synth_long_poisoned, tie_rows
from drive import (check_k4, check_k14, cmp_long, handle, k4_events, k14_events, recognise_dev_np, recognise_long_dev_np,
                   same, tags)
from refs import NTHREADS, get_dis, want_best

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = DIS_ERR = 0xFFFFFFFF
SYM, BAND, SIGN = sr_b200.DTW_SYM_P1, sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN
INT32_MAX = 2 ** 31 - 1
STRIDE = ob.FTR_DTYPE.itemsize
# tags of sr_timing_collect
VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL, DTW_BAND = range(7)
TAG_BLOCKS, TAG_SEGS, TAG_SYM = 11, 12, 14
# two rows whose get_dis is 65 536: squared differences 65 535^2 + 362^2 + 5^2 + 1^2 = 2^32 - 1 (u32), sqrtf -> 2^32
ROW_HI = np.array([32767, 362, 5, 1] + [0] * 8, np.int16)
ROW_LO = np.array([-32768] + [0] * 11, np.int16)


# ---- plain references (CPU) ----------------------------------------------------------------------------------------
def in_band(i, j, I, M, r):
    return 0 <= i < I and 0 <= j < M and abs(j - (i * M) // I) <= r


def sym_ref(x, y, r):
    """g(I-1, M-1) cell by cell from the three predecessor moves, or None when unreachable"""
    I, M = len(x), len(y)
    d = {(i, j): get_dis(x[i], y[j]) for i in range(I) for j in range(M)}
    g = {}
    for i in range(I):
        for j in range(M):
            if not in_band(i, j, I, M, r):
                continue
            if i == j == 0:
                g[0, 0] = 2 * d[0, 0]
                continue
            cand = []
            if (i - 1, j - 2) in g and in_band(i, j - 1, I, M, r):
                cand.append(g[i - 1, j - 2] + 2 * d[i, j - 1] + d[i, j])
            if (i - 1, j - 1) in g:
                cand.append(g[i - 1, j - 1] + 2 * d[i, j])
            if (i - 2, j - 1) in g and in_band(i - 1, j, I, M, r):
                cand.append(g[i - 2, j - 1] + 2 * d[i - 1, j] + d[i, j])
            if cand:
                g[i, j] = min(cand)
    return g.get((I - 1, M - 1))


def all_paths(I, M, r):
    """every P = 1 path from (0, 0) to (I-1, M-1) through the band, as a list of (cell, weight) terms"""
    out = []

    def walk(i, j, terms):
        if (i, j) == (I - 1, M - 1):
            out.append(terms)
            return
        for mid, end in (((i + 1, j + 1), (i + 1, j + 2)), (None, (i + 1, j + 1)), ((i + 1, j + 1), (i + 2, j + 1))):
            if not in_band(*end, I, M, r) or (mid and not in_band(*mid, I, M, r)):
                continue
            walk(*end, terms + ([(end, 2)] if mid is None else [(mid, 2), (end, 1)]))

    if in_band(0, 0, I, M, r):
        walk(0, 0, [((0, 0), 2)])
    return out


def test_oracle_equals_plain_cell_reference():
    """sro_sym == sym_ref on every I, M in 1..12 (the 2:1 guard's rejects included), every r in 0..12 and 118, with tie-heavy
    {0, 1} rows, +-32 767 rows and small random rows"""
    so = ox.sym_oracle()
    rng = np.random.default_rng(0x5A1)
    n = n_err = 0
    for k, (I, M) in enumerate(itertools.product(range(1, 13), range(1, 13))):
        kind = ("tie", "full", "small")[k % 3]
        x, y = tie_rows(rng, I, kind), tie_rows(rng, M, kind)
        bank = sr_b200.make_bank(make_ftr([y]), STRIDE)
        for r in list(range(13)) + [118]:
            got = int(so.dtw_batch(make_ftr([x]), bank, 1, STRIDE, band_r=r)[0, 0])
            g = sym_ref(x, y, r)
            want = DIS_ERR if g is None or I > 2 * M or 2 * I < M else g // (I + M)
            assert got == want, (I, M, r, kind, got, want)
            assert so.g(x, y, r) == g, (I, M, r)
            n += 1
            n_err += got == DIS_ERR
    assert n == 144 * 14 and 0 < n_err < n


def test_brute_force_every_path_weighs_i_plus_m():
    """for I, M <= 7 and r in 0..6: every complete P = 1 path weighs exactly I + M, the cheapest weighted sum is g, and
    the end cell is unreachable exactly when there is no path"""
    so = ox.sym_oracle()
    rng = np.random.default_rng(0x5A2)
    n_paths = n_unreach = 0
    for I, M in itertools.product(range(1, 8), range(1, 8)):
        x, y = tie_rows(rng, I, "small"), tie_rows(rng, M, "small")
        d = {(i, j): get_dis(x[i], y[j]) for i in range(I) for j in range(M)}
        for r in range(7):
            paths = all_paths(I, M, r)
            g = so.g(x, y, r)
            if not paths:
                assert g is None, (I, M, r)
                n_unreach += 1
                continue
            for p in paths:
                assert sum(w for _, w in p) == I + M, (I, M, r, p)
            assert g == min(sum(w * d[c] for c, w in p) for p in paths), (I, M, r)
            n_paths += len(paths)
    assert n_paths > 500 and n_unreach > 20


def planted_band_edge():
    """the first (I, M, r) whose end cell is in the band and reachable when intermediate cells are not checked, but not
    when they are"""
    for I, M in itertools.product(range(2, 12), range(2, 12)):
        if I > 2 * M or 2 * I < M:
            continue
        for r in range(4):
            if not in_band(I - 1, M - 1, I, M, r) or all_paths(I, M, r):
                continue
            reach = {(0, 0)}
            for i in range(I):
                for j in range(M):
                    if in_band(i, j, I, M, r) and {(i - 1, j - 2), (i - 1, j - 1), (i - 2, j - 1)} & reach:
                        reach.add((i, j))
            if (I - 1, M - 1) in reach:
                return I, M, r
    return None


def test_planted_band_edge_scores_dis_err():
    """a pair whose in-band end cell is reachable only through an out-of-band intermediate cell scores SR_DIS_ERR"""
    case = planted_band_edge()
    assert case is not None
    I, M, r = case
    rng = np.random.default_rng(0x5A3)
    x, y = tie_rows(rng, I, "small"), tie_rows(rng, M, "small")
    assert sym_ref(x, y, r) is None and ox.sym_oracle().g(x, y, r) is None
    bank = sr_b200.make_bank(make_ftr([y]), STRIDE)
    assert int(ox.sym_oracle().dtw_batch(make_ftr([x]), bank, 1, STRIDE, band_r=r)[0, 0]) == DIS_ERR
    assert sym_ref(x, y, r + 1) is not None or not in_band(I - 1, M - 1, I, M, r + 1)


def test_headroom_every_get_dis_65536():
    """I = M = 119 with every get_dis 65 536: g = 238 * 65 536, score 65 536"""
    assert get_dis(ROW_HI, ROW_LO) == 65536
    x, y = np.tile(ROW_HI, (119, 1)), np.tile(ROW_LO, (119, 1))
    so = ox.sym_oracle()
    assert so.g(x, y, 118) == 238 * 65536
    bank = sr_b200.make_bank(make_ftr([y]), STRIDE)
    assert int(so.dtw_batch(make_ftr([x]), bank, 1, STRIDE, band_r=118)[0, 0]) == 65536


# ---- sr_dtw_batch (GPU) --------------------------------------------------------------------------------------------
RADII = list(range(21)) + [30, 60, 117, 118, INT32_MAX]


@pytest.mark.gpu
@pytest.mark.parametrize("T", (1, 31, 32, 33, 80, 200))
def test_dtw_batch_sym_equals_oracle(T):
    """score, best_idx and best_dis of sr_dtw_batch(SR_DTW_SYM_P1[, CHECK_SIGN]) bit for bit against the oracle: every
    radius of RADII, inputs of 0..120 frames (every I in 1..119 over the widths, and the 2:1 edges), planted slots"""
    so = ox.sym_oracle()
    rng = np.random.default_rng(0x5B0 + T)
    bank = bank_planted(rng, T)
    M = bank.view(np.uint16)[:, 1].astype(np.int64)
    frms = [0, 120, 1, 119] + [int(m) * 2 for m in M[:4] if 0 < m <= 59] + [(int(m) + 1) // 2 for m in M[:4] if 0 < m <= 119]
    frms += [int(x) for x in rng.integers(1, 120, 40 - len(frms))]
    fin = inputs(rng, frms)
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    try:
        for r in RADII if T in (33, 80) else (0, 1, 10, 16, 118, INT32_MAX):
            for flags in (SYM, SYM | SIGN):
                want = so.dtw_batch(fin, bank, T, 4096, check_sign=flags & SIGN, band_r=r, nthreads=NTHREADS)
                score, bi, bd = h.dtw(fin, flags=flags, band_r=r)
                assert np.array_equal(score, want), (T, r, flags, np.argwhere(score != want)[:4].tolist())
                wi, wd = want_best(want)
                assert np.array_equal(bi, wi) and np.array_equal(bd, wd), (T, r, flags)
                s2, bi2, bd2 = h.dtw(fin, flags=flags, band_r=r, want_score=False)     # score NULL
                assert s2 is None and np.array_equal(bi2, wi) and np.array_equal(bd2, wd)
            assert (want[:2] == DIS_ERR).all()                                   # frm_num 0 and 120 inputs
    finally:
        h.close()


@pytest.mark.gpu
def test_dtw_batch_sym_headroom_and_band_edge():
    """the 65 536 headroom case scores 65 536 and the planted band-edge pair SR_DIS_ERR on the GPU too"""
    h = sr_b200.Handle(0)
    try:
        fin = make_ftr([np.tile(ROW_HI, (119, 1))])
        h.set_bank(sr_b200.make_bank(make_ftr([np.tile(ROW_LO, (119, 1))]), 4096), 1, 4096)
        for r in (16, 118, INT32_MAX):
            assert int(h.dtw(fin, SYM, r)[0][0, 0]) == 65536
        I, M, r = planted_band_edge()
        rng = np.random.default_rng(0x5A3)
        x, y = tie_rows(rng, I, "small"), tie_rows(rng, M, "small")
        h.set_bank(sr_b200.make_bank(make_ftr([y]), 4096), 1, 4096)
        assert int(h.dtw(make_ftr([x]), SYM, r)[0][0, 0]) == DIS_ERR
        assert int(h.dtw(make_ftr([x]), SYM, r + 1)[0][0, 0]) == int(ox.sym_oracle().dtw_batch(
            make_ftr([x]), sr_b200.make_bank(make_ftr([y]), 4096), 1, 4096, band_r=r + 1)[0, 0])
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("B", (2111, 2112, 2113, 4225))
def test_dtw_batch_sym_grid_boundaries(B):
    """batches around one grid pass (132 CTAs x 16 warps = 2 112 inputs per tile column) and two, best-only calls"""
    so = ox.sym_oracle()
    rng = np.random.default_rng(0x5C0 + B)
    T = 32
    fin = inputs(rng, [int(x) for x in rng.integers(8, 24, B)])
    bank = sr_b200.make_bank(inputs(rng, [int(x) for x in rng.integers(8, 24, T)]), 4096)
    want = so.dtw_batch(fin, bank, T, 4096, band_r=6, nthreads=NTHREADS)
    h = sr_b200.Handle(0)
    try:
        h.set_bank(bank, T, 4096)
        score, bi, bd = h.dtw(fin, SYM, 6)
        assert np.array_equal(score, want)
        _, bi2, bd2 = h.dtw(fin, SYM, 6, want_score=False)
        wi, wd = want_best(want)
        assert np.array_equal(bi, wi) and np.array_equal(bd, wd) and np.array_equal(bi2, wi) and np.array_equal(bd2, wd)
    finally:
        h.close()


# ---- the setter rules (GPU: the calls need a handle) ----------------------------------------------------------------
@pytest.mark.gpu
def test_set_match_rules_and_sym_band_refused():
    """sr_set_match(SR_DTW_SYM_P1, r) takes any r >= 0 and round-trips; SYM | BAND, other bits and r < 0 fail and leave
    the setting unchanged; sr_dtw_batch with SYM | BAND fails and writes nothing"""
    h = sr_b200.Handle(0)
    try:
        for r in (0, 5, 118, INT32_MAX):
            h.set_match(SYM, r)
            assert h.match() == (SYM, r)
        h.set_match(SYM, 7)
        for flags, r in ((SYM | BAND, 3), (SYM | SIGN, 3), (SYM | 8, 3), (8, 0), (BAND | 4, 3), (SYM, -1)):
            with pytest.raises(sr_b200.SrError):
                h.set_match(flags, r)
            assert h.match() == (SYM, 7)
        rng = np.random.default_rng(0x5D0)
        h.set_bank(bank_planted(rng, 8), 8, 4096)
        fin = inputs(rng, [30, 40, 50])
        score = np.full((3, 8), 0xA5A5A5A5, np.uint32)
        bi, bd = np.full(3, 0xA5A5A5A5, np.uint32), np.full(3, 0xA5A5A5A5, np.uint32)
        c0 = h.launch_count()
        for flags in (SYM | BAND, SYM | BAND | SIGN):
            with pytest.raises(sr_b200.SrError):
                h._ck(sr_b200.lib().sr_dtw_batch(h._h, sr_b200._p(fin), 3, flags, 4, sr_b200._p(score), sr_b200._p(bi),
                                                  sr_b200._p(bd)))
        assert h.launch_count() == c0
        assert (score == 0xA5A5A5A5).all() and (bi == 0xA5A5A5A5).all() and (bd == 0xA5A5A5A5).all()
        import torch
        dev = torch.device("cuda:0")
        d_in = torch.from_numpy(fin.view(np.uint8).copy()).to(dev)
        d_out = [torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device=dev) for n in (24, 3, 3)]
        with pytest.raises(sr_b200.SrError):
            h.dtw_dev(d_in.data_ptr(), 3, SYM | BAND, 4, *[t.data_ptr() for t in d_out])
        h.sync()
        assert h.launch_count() == c0 and all((t == 0x5A5A5A5A).all().item() for t in d_out)
    finally:
        h.close()


# ---- recognition under the sym matcher -------------------------------------------------------------------------------
U = 16000
PLANTED = [0, 1, 1047, 1048, 1049, 2096, 3199]


def _tpl_bank(slots, valid):
    tpl = sr_b200.synth_pcm_host(8, 8000, 0x7E3A0000)
    ob.plant_sample0(tpl, [1, 4], 0x7E3A)
    e = ob.recognise_pinned(ob.best_oracle(), tpl, 2400, None, 0, 4096)
    assert (e["status"] == 0).all()
    return sr_b200.make_bank(e["ftr"][slots], valid=valid)


@pytest.fixture(scope="module")
def case():
    """3 200 two-second utterances (four 1 048-utterance chunks of the host call, so the packed transport engages), a
    silent one, one over 119 frames, planted segments from sample 0; a 20-slot bank with duplicates and unsigned slots"""
    ora = ob.best_oracle()
    B = 3200
    pcm = sr_b200.synth_pcm_host(B, U, 0x5E5E0000, 2)
    rng = np.random.default_rng(0x5E)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    ob.plant_sample0(pcm, PLANTED, 0x5E)
    front = ob.recognise_pinned(ora, pcm, 2400, None, 0, 4096)
    assert front["status"][3] == 1 and front["status"][4] == 2
    slots = list(range(8)) + [0, 2, 5, 5, 1, 7, 3, 3, 6, 4, 0, 2]
    valid = [1] * 20
    valid[3] = valid[9] = 0
    return {"pcm": pcm, "front": front, "bank": _tpl_bank(slots, valid)}


@pytest.mark.gpu
@pytest.mark.parametrize("r", (4, 16, 118))
def test_recognise_sym_equals_oracle_composition(case, r):
    """set_match(SR_DTW_SYM_P1, r): the host call on the plain and the packed transport, sr_recognise_batch_dev on a torch
    stream, and sr_recognise_batch_multi over two handles (on two devices when two are visible) all equal the oracle"""
    import torch
    pcm, front, bank = case["pcm"], case["front"], case["bank"]
    want = ox.compose_recognise(front, bank, 20, SYM, r)
    assert (want["best_dis"][want["status"] == 0] != NULL).sum() > 1500
    h = handle(bank, 20, SYM, r)
    try:
        h.set_transport(0)
        same(h.recognise(pcm, 2400), want, "host plain")
        h.set_transport(1)
        same(h.recognise(pcm, 2400), want, "host packed")
        assert h.transport_stats()[0] > 0
        same(recognise_dev_np(h, pcm, 2400, 20), want, "device launch on a torch stream")
        h.use_own_stream()
        h2 = sr_b200.Handle(1 if torch.cuda.device_count() > 1 else 0)
        h2.set_bank(bank, 20, 4096)
        h2.set_match(SYM, r)
        same(sr_b200.recognise_multi([h, h2], pcm, 2400, want=sr_b200.RECOG_FIELDS), want, "multi")
        h2.close()
    finally:
        h.close()


@pytest.mark.gpu
def test_geom_b_recognise_sym_equals_own_oracle():
    """GEOM_B features (parity unpinned) under the sym matcher: the port's GEOM_B front end, then tests/oracle_ext/sym.c"""
    po = ob.port()
    h = sr_b200.Handle(0)
    try:
        h.set_geometry(1)
        T = 6
        bank, est = h.enrol(sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000), 2400)
        assert (est == 0).all()
        h.set_bank(bank, T, 4096)
        h.set_match(SYM, 16)
        pcm = sr_b200.synth_pcm_host(128, 8000, 0x5EED0000)
        ob.plant_sample0(pcm, [0, 5, 127], 0xB5)
        front = ob.recognise_pinned(po, pcm, 2400, None, 0, 4096, geom_b=True)
        want = ox.compose_recognise(front, bank, T, SYM, 16)
        same(h.recognise(pcm, 2400), want, "GEOM_B")
        assert (want["status"] == 0).sum() > 100
    finally:
        h.close()


@pytest.mark.gpu
def test_mixed_matchers_are_refused_by_multi_and_groups(case):
    """sr_recognise_batch_multi and a stream group of two handles on one device refuse sym beside greedy, band at the same
    radius and sym at another radius, and run once the matchers agree"""
    bank, pcm = case["bank"], case["pcm"][:64]
    for second in ((0, 0), (BAND, 16), (SYM, 15)):
        a, b = handle(bank, 20, SYM, 16), handle(bank, 20, *second)
        try:
            with pytest.raises(sr_b200.SrError):
                sr_b200.recognise_multi([a, b], pcm, 2400)
            pool = sr_b200.StreamPool([a, b], 8, 8000, 2400)
            with pytest.raises(sr_b200.SrError):
                pool.push(np.ascontiguousarray(pcm[:8, :800]))
            b.set_match(SYM, 16)
            pool.push(np.ascontiguousarray(pcm[:8, :800]))
            pool.close()
            out = sr_b200.recognise_multi([a, b], pcm, 2400)
            assert np.array_equal(out["score"], a.recognise(pcm, 2400)["score"])
        finally:
            a.close()
            b.close()


# ---- streaming: the K4 pool and group -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("arrival,group", [("lockstep", False), ("ragged", False), ("ragged", True)],
                         ids=["lockstep", "ragged", "group_of_two"])
def test_k4_streams_sym_equal_oracle(case, arrival, group):
    """fixed-capture stream pushes under the sym matcher: every event equals the oracle's get_mfcc of its segment, then
    tests/oracle_ext/sym.c and the argmin"""
    S, L, T = 24, 40000, 20
    bank = case["bank"]
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDD000, 3)
    pcm[3] = 2048
    hs = [handle(bank, T, SYM, 16) for _ in range(2 if group else 1)]
    try:
        pool = sr_b200.StreamPool(hs if group else hs[0], S, L, 2400)
        events = k4_events(pool, pcm, arrival, np.random.default_rng(0x5F))
        check_k4(events, pool, pcm, bank, T, (SYM, 16))
        pool.close()
    finally:
        for h in hs:
            h.close()


MATCHERS = ((0, 0), (SYM, 16), (BAND, 16))          # greedy -> sym -> band, switched between pushes


@pytest.mark.gpu
def test_k4_matcher_switched_between_pushes(case):
    """greedy -> sym -> band -> ... between the pushes of one K4 pool: each event equals the oracle under the matcher of
    its push"""
    S, L, T = 16, 40000, 20
    bank = case["bank"]
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDE000, 3)
    h = handle(bank, T, 0, 0)
    try:
        pool = sr_b200.StreamPool(h, S, L, 2400)

        def on_push(p):
            m = MATCHERS[p % 3]
            h.set_match(*m)
            return m
        events = k4_events(pool, pcm, "lockstep", None, on_push)
        assert {m for _, m in events} == set(MATCHERS)
        check_k4(events, pool, pcm, bank, T)
        pool.close()
    finally:
        h.close()


# ---- long recordings and live long streams --------------------------------------------------------------------------
@pytest.mark.gpu
def test_long_batch_and_dev_sym_equal_oracle():
    """sr_recognise_long_batch and its _dev form under SR_DTW_SYM_P1 equal the composed oracle on ragged recordings"""
    lens = np.array([70001, 161, 123457, 99999, 200000], np.uint32)
    pcm = synth_long_poisoned(lens, 200000, 0x5F10)
    bank, T = ox.synth_bank()
    h = handle(bank, T, SYM, 10)
    try:
        want = ox.recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, T, 4096, 64, lens, match=(SYM, 10))
        assert sum((want["segs"][b, :int(want["n_segs"][b])]["best_dis"] != NULL).sum() for b in range(len(lens))) > 20
        cmp_long(h.recognise_long_batch(pcm, 64, 2400, lens), want)
        cmp_long(recognise_long_dev_np(h, pcm, lens, 64), want)
    finally:
        h.close()


@pytest.mark.gpu
def test_k14_long_streams_sym_equal_oracle():
    """a live long-stream pool under the sym matcher: every closed segment's event equals the composed oracle"""
    xs = list(ox.synth_long(6, 120000, 0x5F20))
    xs[2] = xs[2][:50000]
    bank, T = ox.synth_bank()
    h = handle(bank, T, SYM, 16)
    try:
        pool = sr_b200.LongStreamPool(h, len(xs), 4000, 2400)
        events = k14_events(pool, xs, 4000)
        pool.close()
        check_k14(events, xs, bank, T, [(SYM, 16)])
    finally:
        h.close()


@pytest.mark.gpu
def test_k14_matcher_switched_between_pushes():
    """greedy -> sym -> band between the pushes of one live long-stream pool: each event equals the oracle under the
    matcher of the push that returned it"""
    xs = list(ox.synth_long(4, 160000, 0x5F30))
    bank, T = ox.synth_bank()
    h = handle(bank, T, 0, 0)
    try:
        pool = sr_b200.LongStreamPool(h, len(xs), 3000, 2400)

        def on_push(p):
            m = MATCHERS[p % 3]
            h.set_match(*m)
            return m
        events = k14_events(pool, xs, 3000, on_push)
        pool.close()
        assert {m for _, m in events} == set(MATCHERS)
        check_k14(events, xs, bank, T, list(MATCHERS))
    finally:
        h.close()


# ---- launch accounting ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_tag_14_where_tag_6_is_under_the_band_matcher(case):
    """the recognise, long-recognise and sr_dtw_batch calls under SYM launch what they launch under BAND, with tag 14 in
    place of tag 6, for r on both sides of every band-kernel choice"""
    pcm, bank = case["pcm"][:64], case["bank"]
    lpcm = ox.synth_long(3, 100000, 0x5F40)
    fin = case["front"]["ftr"][:64]
    h = handle(bank, 20, 0, 0)
    try:
        h.set_transport(0)
        h.timing_enable(4096)
        for r in (10, 15, 16, 118):
            runs = {}
            for flags in (BAND, SYM):
                h.set_match(flags, r)
                c0 = h.launch_count()
                h.recognise(pcm, 2400)
                h.recognise_long_batch(lpcm, 32, 2400)
                h.dtw(fin, flags | SIGN, r)
                runs[flags] = (h.launch_count() - c0, tags(h))
            nb, tb = runs[BAND]
            ns, ts = runs[SYM]
            assert ns == nb and ts == [TAG_SYM if t == DTW_BAND else t for t in tb], r
            assert ts.count(TAG_SYM) == 3 and DTW_BAND not in ts and DTW not in ts
        assert ts[:6] == [VAD_, MFCC_, STATUS, BEST_INIT, TAG_SYM, BEST_FINAL]
    finally:
        h.close()


# ---- concurrency ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_threads_under_sym_band_and_greedy(case):
    """handles under sym, band and greedy (recognise and long recognise) run on threads released by one barrier; every
    repetition equals its serial run"""
    pcm, bank = case["pcm"][:256], case["bank"]
    lpcm = ox.synth_long(3, 120000, 0x5F50)
    jobs = []
    for flags, r in ((SYM, 16), (SYM, 4), (BAND, 16), (0, 0)):
        jobs.append((flags, r, "short"))
        jobs.append((flags, r, "long"))
    handles = [handle(bank, 20, f, r) for f, r, _ in jobs]

    def run_job(i):
        h, kind = handles[i], jobs[i][2]
        if kind == "short":
            return h.recognise(pcm, 2400)
        return h.recognise_long_batch(lpcm, 32, 2400)

    try:
        serial = [run_job(i) for i in range(len(jobs))]
        want = ox.compose_recognise({k: v[:256] for k, v in case["front"].items()}, bank, 20, SYM, 16)
        same(serial[0], want, "serial sym")
        barrier = threading.Barrier(len(jobs))
        results = [[None] * 3 for _ in jobs]
        errors = []

        def run(i):
            try:
                barrier.wait()
                for rep in range(3):
                    results[i][rep] = run_job(i)
            except Exception as e:                      # noqa: BLE001
                errors.append(e)
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        for i in range(len(jobs)):
            for rep in range(3):
                for k, v in serial[i].items():
                    assert np.asarray(results[i][rep][k]).tobytes() == np.asarray(v).tobytes(), (jobs[i], rep, k)
    finally:
        for h in handles:
            h.close()


# ---- real speech, reported ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_real_speech_sym_reported():
    """enrol each digit recording's segments (template k in slot 4k) and recognise its twin with sr_recognise_long_batch
    under greedy, band r = 118 and sym r = 118: decisions equal the oracle; segments whose command equals their position
    are printed, not asserted"""
    port = ob.port()
    h = sr_b200.Handle(0)
    try:
        for a_name, b_name in real_speech_pairs():
            a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
            h.set_match(0, 0)
            h.set_bank(np.zeros((0, 4096), np.uint8), 0, 4096)
            ea = h.recognise_long_batch(a[None], 32, 2400)
            ma = int(ea["n_segs"][0])
            ftr = ox.ftr_of_segments(port, a[None], ea["atap"], [(0, int(s["start"]), int(s["end"]) if s["end"] != NULL
                                                                   else int(s["start"])) for s in ea["segs"][0, :ma]])
            ftr4 = np.zeros(4 * ma, ob.FTR_DTYPE)
            ftr4[0::4] = ftr
            valid = np.zeros(4 * ma, bool)
            valid[0::4] = True
            bank, T = sr_b200.make_bank(ftr4, 4096, valid), 4 * ma
            h.set_bank(bank, T, 4096)
            line = []
            for flags, r, name in ((0, 0, "greedy"), (BAND, 118, "band r=118"), (SYM, 118, "sym r=118")):
                h.set_match(flags, r)
                got = h.recognise_long_batch(b[None], 32, 2400)
                want = ox.recognise_long(ox.long_oracle(), port, b[None], 2400, bank, T, 4096, 32, match=(flags, r))
                cmp_long(got, want)
                m = min(int(got["n_segs"][0]), ma)
                right = int((got["segs"][0, :m]["cmd"] == np.arange(m)).sum())
                line.append("%s %d/%d" % (name, right, m))
            print("%s -> %s: %s" % (a_name, b_name, ", ".join(line)))
    finally:
        h.close()
