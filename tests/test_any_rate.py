"""The banded DP without the 2:1 length guard (SR_DTW_BAND | SR_DTW_ANY_RATE, an extension the reference does not have;
parity unpinned) in sr_dtw_batch and as the matcher of every recognition call (sr_set_match).

CPU: the header and the binding define the bit; the C oracle (tests/oracle_ext/rate.c) equals a plain Python DP on every shape
up to 12 x 12 and the oracle port's SR_DTW_BAND DP on every pair within 2:1; it reproduces the real-speech accuracy of the
four digit recordings. GPU: the setter and flag rules; sr_dtw_batch equals the oracle bit for bit on every (I, M) in
1..119 x 1..119 at radii that pick each band kernel, and plain SR_DTW_BAND on every pair within 2:1; every recognition
path under the matcher equals the oracle composition, and a bank of stretched and shrunk templates makes the guard change
decisions; bytes written and timing tags are the band matcher's; real speech, reported.
sr_recognise_batch_dev_allgather is not run here: it needs two NCCL ranks. Every GPU test makes its own handles."""
import itertools
import os
import re

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from test_extension_refs import NTHREADS
from test_sym_match import (DIGITS, INT32_MAX, _bank_planted, _cmp_long, _ftr, _inputs, _k14_events, _k4_events, _rows,
                            _same, _want_best, get_dis)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = DIS_ERR = 0xFFFFFFFF
BAND, SIGN, SYM, ANY = sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN, sr_b200.DTW_SYM_P1, sr_b200.DTW_ANY_RATE
RATE = BAND | ANY
STRIDE = ob.FTR_DTYPE.itemsize
KERNEL_RADII = (0, 1, 10, 15, 16, 40, 118)           # warp-scan (<= 15), thread form (10), whole row (>= 16)
# tags of sr_timing_collect
VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL, DTW_BAND = range(7)


def guard_ok(I, M):
    return not (I > 2 * M or 2 * I < M)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_header_and_binding_define_the_bit():
    with open(os.path.join(ROOT, "include", "speech_recog.h")) as f:
        m = re.search(r"#define\s+SR_DTW_ANY_RATE\s+(\w+)", f.read())
    assert m and int(m.group(1).rstrip("uU"), 0) == 8
    assert sr_b200.DTW_ANY_RATE == 8 and len({BAND, SIGN, SYM, ANY}) == 4


def rate_ref(x, y, r):
    """D(I-1, M-1) of the band DP, cell by cell, without any length guard, or None when unreachable"""
    I, M = len(x), len(y)
    D = {}
    for i in range(I):
        for j in range(M):
            if abs(j - (i * M) // I) > r:
                continue
            prev = [D[c] for c in ((i - 1, j), (i, j - 1), (i - 1, j - 1)) if c in D]
            if i == j == 0:
                prev = [0]
            if prev:
                D[i, j] = min(prev) + get_dis(x[i], y[j])
    return D.get((I - 1, M - 1))


def test_oracle_equals_plain_reference_on_every_small_shape():
    """sro_rate == rate_ref on every I, M in 1..12 (ratios up to 12:1 both ways) at every r in 0..12 and 118, and the end
    cell outside the band (ceil(M/I) - 1 > r) always scores SR_DIS_ERR"""
    ro = ox.rate_oracle()
    rng = np.random.default_rng(0xA11)
    n_far = n_err = 0
    for k, (I, M) in enumerate(itertools.product(range(1, 13), range(1, 13))):
        kind = ("tie", "full", "small")[k % 3]
        x, y = _rows(rng, I, kind), _rows(rng, M, kind)
        bank = sr_b200.make_bank(_ftr([y]), STRIDE)
        for r in list(range(13)) + [118]:
            d = rate_ref(x, y, r)
            assert ro.d(x, y, r) == d, (I, M, r)
            got = int(ro.dtw_batch(_ftr([x]), bank, 1, STRIDE, band_r=r)[0, 0])
            assert got == (DIS_ERR if d is None else d // (I + M)), (I, M, r)
            if M > I and -(-M // I) - 1 > r:
                assert got == DIS_ERR
            n_far += not guard_ok(I, M) and got != DIS_ERR
            n_err += got == DIS_ERR
    assert n_far > 500 and n_err > 100


def test_oracle_equals_band_oracle_within_the_guard():
    """on every pair of 1..119-frame sets within 2:1 (sampled per shape) the new oracle scores what the port's SR_DTW_BAND
    DP scores at the same r; outside 2:1 the port says SR_DIS_ERR and the new oracle scores every pair at r = 118"""
    ro, po = ox.rate_oracle(), ob.port()
    rng = np.random.default_rng(0xA12)
    frms = [1, 2, 3, 59, 60, 61, 118, 119] + [int(v) for v in rng.integers(1, 120, 24)]
    fin = _inputs(rng, frms)
    bank = sr_b200.make_bank(_inputs(rng, frms[::-1]), 4096)
    I = np.array(frms)[:, None]
    M = np.array(frms[::-1])[None, :]
    inside = (I <= 2 * M) & (M <= 2 * I)
    for r in (0, 1, 5, 10, 15, 16, 40, 118):
        want, _ = po.dtw_batch(fin, bank, len(frms), 4096, band_r=r, nthreads=NTHREADS)
        got = ro.dtw_batch(fin, bank, len(frms), 4096, band_r=r, nthreads=NTHREADS)
        assert np.array_equal(got[inside], want[inside]), r
        assert (want[~inside] == DIS_ERR).all()
        if r == 118:
            assert (got != DIS_ERR).all()


def _real_speech_pairs():
    return ((DIGITS[0], DIGITS[1]), (DIGITS[1], DIGITS[0]), (DIGITS[2], DIGITS[3]), (DIGITS[3], DIGITS[2]))


def _digit_bank(port, lo, a):
    """template k = segment k of recording a, in slot 4k (the other slots unsigned)"""
    ea = ox.recognise_long(lo, port, a[None], 2400, None, 0, 4096, 32)
    ma = int(ea["n_segs"][0])
    ftr = ox.ftr_of_segments(port, a[None], ea["atap"], [(0, int(s["start"]), int(s["end"]) if s["end"] != NULL
                                                          else int(s["start"])) for s in ea["segs"][0, :ma]])
    ftr4 = np.zeros(4 * ma, ob.FTR_DTYPE)
    ftr4[0::4] = ftr
    valid = np.zeros(4 * ma, bool)
    valid[0::4] = True
    return sr_b200.make_bank(ftr4, 4096, valid), 4 * ma, ma


def test_real_speech_accuracy_on_the_oracles():
    """the digit recordings, each recognised against its twin's segments at r = 118: the band DP gets 6, 8, 3, 3 right
    (20 of 46), the same DP without the guard 4, 8, 9, 8 (29 of 46). A fixed computation on fixed data, not a claim about
    speech in general"""
    lo, port = ox.long_oracle(), ob.port()
    got = []
    for a_name, b_name in _real_speech_pairs():
        a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
        bank, T, ma = _digit_bank(port, lo, a)
        row = []
        for flags in (BAND, RATE):
            w = long_oracle(b[None], bank, T, flags, 118, 32)
            m = min(int(w["n_segs"][0]), ma)
            row.append(int((w["segs"][0, :m]["cmd"] == np.arange(m)).sum()))
        got.append(tuple(row) + (ma,))
    assert got == [(6, 4, 10), (8, 8, 10), (3, 9, 13), (3, 8, 13)], got


# ---- oracle compositions -----------------------------------------------------------------------------------------------
def _scores(ftr, bank, T, flags, r):
    """the oracle's template scan under a matcher (0 greedy, BAND, RATE) with the save_sign check"""
    if flags == RATE:
        return ox.rate_oracle().dtw_batch(ftr, bank, T, 4096, check_sign=1, band_r=r, nthreads=NTHREADS)
    return ob.port().dtw_batch(ftr, bank, T, 4096, check_sign=1, band_r=r if flags else -1, nthreads=NTHREADS)[0]


def _compose(front, bank, T, flags, r):
    """the front end, then the scan under the matcher, the strict '<' first-wins argmin, cmd = idx / 4"""
    out = {k: front[k].copy() for k in ("atap", "seg_off", "ftr", "status")}
    B = len(out["status"])
    out["score"] = np.full((B, T), NULL, np.uint32)
    out["best_idx"], out["best_dis"], out["cmd"] = np.zeros(B, np.uint32), np.full(B, NULL, np.uint32), np.zeros(B, np.uint32)
    good = out["status"] == 0
    sc = _scores(out["ftr"][good], bank, T, flags, r)
    out["score"][good] = sc
    i = np.argmin(sc, axis=1)
    out["best_idx"][good] = i
    out["best_dis"][good] = sc[np.arange(len(i)), i]
    out["cmd"][good] = i // 4
    return out


def long_oracle(pcm, bank, T, flags, r, max_segs, lens=None):
    """sr_recognise_long_batch composed from the oracles: the long-form VAD and front end, the scan under the matcher"""
    lo, port = ox.long_oracle(), ob.port()
    if flags != RATE:
        return ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, max_segs, lens, band_r=r if flags else -1)
    want = ox.recognise_long(lo, port, pcm, 2400, bank, 0, 4096, max_segs, lens)
    segs = want["segs"]
    todo = [(b, k) for b in range(len(segs)) for k in range(min(int(want["n_segs"][b]), max_segs)) if segs[b, k]["status"] == 0]
    if todo and T:
        ftr = ox.ftr_of_segments(port, pcm, want["atap"], [(b, int(segs[b, k]["start"]), int(segs[b, k]["end"]))
                                                            for b, k in todo])
        sc = _scores(ftr, bank, T, RATE, r)
        for i, (b, k) in enumerate(todo):
            j = int(np.argmin(sc[i]))
            if sc[i, j] != NULL:
                segs[b, k]["best_idx"], segs[b, k]["best_dis"], segs[b, k]["cmd"] = j, sc[i, j], j // 4
    return want


# ---- sr_dtw_batch (GPU) ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_match_and_flag_rules():
    """BAND | ANY_RATE at r = 0, 10, 15, 16, 118, 1000 round-trips through sr_get_match; ANY_RATE alone, with SYM, with
    SYM | BAND, and r < 0 fail and leave the setting unchanged; sr_dtw_batch and its _dev form refuse the same flags with
    no launch and no output byte written"""
    h = sr_b200.Handle(0)
    try:
        for r in (0, 10, 15, 16, 118, 1000):
            h.set_match(RATE, r)
            assert h.match() == (RATE, r)
        h.set_match(RATE, 7)
        bad = ((ANY, 3), (ANY | SYM, 3), (ANY | SYM | BAND, 3), (RATE, -1), (RATE | SIGN, 3))
        for flags, r in bad:
            with pytest.raises(sr_b200.SrError):
                h.set_match(flags, r)
            assert h.match() == (RATE, 7)
        rng = np.random.default_rng(0xA20)
        h.set_bank(_bank_planted(rng, 8), 8, 4096)
        fin = _inputs(rng, [30, 40, 50])
        score = np.full((3, 8), 0xA5A5A5A5, np.uint32)
        bi, bd = np.full(3, 0xA5A5A5A5, np.uint32), np.full(3, 0xA5A5A5A5, np.uint32)
        c0 = h.launch_count()
        for flags, r in ((ANY, 3), (ANY | SIGN, 3), (ANY | SYM, 3), (ANY | SYM | BAND, 3), (ANY | SYM | SIGN, 3),
                         (RATE, -1), (RATE | SIGN, -1)):
            with pytest.raises(sr_b200.SrError):
                h._ck(sr_b200.lib().sr_dtw_batch(h._h, sr_b200._p(fin), 3, flags, r, sr_b200._p(score), sr_b200._p(bi),
                                                  sr_b200._p(bd)))
        assert h.launch_count() == c0
        assert (score == 0xA5A5A5A5).all() and (bi == 0xA5A5A5A5).all() and (bd == 0xA5A5A5A5).all()
        import torch
        dev = torch.device("cuda:0")
        d_in = torch.from_numpy(fin.view(np.uint8).copy()).to(dev)
        d_out = [torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device=dev) for n in (24, 3, 3)]
        c1 = h.launch_count()
        for flags in (ANY, ANY | SYM, ANY | SYM | BAND):
            with pytest.raises(sr_b200.SrError):
                h.dtw_dev(d_in.data_ptr(), 3, flags, 4, *[t.data_ptr() for t in d_out])
        h.sync()
        assert h.launch_count() == c1 and all((t == 0x5A5A5A5A).all().item() for t in d_out)
    finally:
        h.close()


def _every_shape_case(kind, seed):
    """inputs of 1..119 frames against a 119-slot bank of 119..1 frames: every (I, M) in 1..119 x 1..119 once"""
    rng = np.random.default_rng(seed)
    frms = list(range(1, 120))
    fin = _ftr([_rows(rng, f, kind) for f in frms])
    bank = sr_b200.make_bank(_ftr([_rows(rng, f, kind) for f in frms[::-1]]), 4096)
    return fin, bank


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("small", "tie"))
def test_dtw_batch_every_shape_equals_oracle(kind):
    """score, best_idx and best_dis of sr_dtw_batch(BAND | ANY_RATE) on every (I, M) in 1..119 x 1..119 (1:119 and 119:1
    included) at every radius that picks a band kernel, bit for bit against the oracle; tie-heavy {0, 1} rows as a second
    case. Every pair within 2:1 scores what plain SR_DTW_BAND scores; outside it BAND says SR_DIS_ERR"""
    ro = ox.rate_oracle()
    fin, bank = _every_shape_case(kind, 0xA30 + (kind == "tie"))
    I = np.arange(1, 120)[:, None]
    M = np.arange(119, 0, -1)[None, :]
    inside = (I <= 2 * M) & (M <= 2 * I)
    h = sr_b200.Handle(0)
    h.set_bank(bank, 119, 4096)
    try:
        for r in KERNEL_RADII:
            want = ro.dtw_batch(fin, bank, 119, 4096, band_r=r, nthreads=NTHREADS)
            score, bi, bd = h.dtw(fin, flags=RATE, band_r=r)
            assert np.array_equal(score, want), (kind, r, np.argwhere(score != want)[:4].tolist())
            wi, wd = _want_best(want)
            assert np.array_equal(bi, wi) and np.array_equal(bd, wd), (kind, r)
            s2, bi2, bd2 = h.dtw(fin, flags=RATE, band_r=r, want_score=False)
            assert s2 is None and np.array_equal(bi2, wi) and np.array_equal(bd2, wd), (kind, r)
            plain, _, _ = h.dtw(fin, flags=BAND, band_r=r)
            assert np.array_equal(plain[inside], score[inside]) and (plain[~inside] == DIS_ERR).all(), (kind, r)
            if r == 118:
                assert (score != DIS_ERR).all()
            assert (score[~inside] != DIS_ERR).any(), r                  # the guard's rejects now score somewhere
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", (1, 33, 80))
def test_dtw_batch_planted_slots_equal_oracle(T):
    """banks with erased, unsigned, frm_num 0 and frm_num 120 slots; inputs of 0..120 frames; with and without
    CHECK_SIGN, at every kernel radius and INT32_MAX"""
    ro = ox.rate_oracle()
    rng = np.random.default_rng(0xA40 + T)
    bank = _bank_planted(rng, T)
    frms = [0, 120, 1, 119, 2, 118, 3, 100] + [int(x) for x in rng.integers(1, 120, 32)]
    fin = _inputs(rng, frms)
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    try:
        for r in KERNEL_RADII + (INT32_MAX,):
            for flags in (RATE, RATE | SIGN):
                want = ro.dtw_batch(fin, bank, T, 4096, check_sign=flags & SIGN, band_r=r, nthreads=NTHREADS)
                score, bi, bd = h.dtw(fin, flags=flags, band_r=r)
                assert np.array_equal(score, want), (T, r, flags, np.argwhere(score != want)[:4].tolist())
                wi, wd = _want_best(want)
                assert np.array_equal(bi, wi) and np.array_equal(bd, wd), (T, r, flags)
            assert (want[:2] == DIS_ERR).all()
    finally:
        h.close()


# ---- recognition under the matcher (GPU) -------------------------------------------------------------------------------
U = 16000
PLANTED = [0, 1, 1047, 1048, 1049, 2096, 3199]


def _stretched_bank():
    """8 synthetic templates, each also shrunk to every third row and stretched to three copies of each row (capped at
    119): 24 slots, command = slot / 4 as usual, one unsigned slot"""
    tpl = sr_b200.synth_pcm_host(8, 8000, 0x7E3A0000)
    e = ob.recognise_pinned(ob.best_oracle(), tpl, 2400, None, 0, 4096)
    assert (e["status"] == 0).all()
    rows = []
    for f in e["ftr"]:
        x = f["mfcc_dat"][:int(f["frm_num"]) * 12].reshape(-1, 12)
        rows += [x, x[::3], np.repeat(x, 3, axis=0)[:119]]
    valid = np.ones(24, bool)
    valid[5] = False
    return sr_b200.make_bank(_ftr(rows), 4096, valid), 24


@pytest.fixture(scope="module")
def case():
    """3 200 two-second utterances (the packed transport engages), a silent one, one over 119 frames, planted segments
    from sample 0; the stretched bank"""
    B = 3200
    pcm = sr_b200.synth_pcm_host(B, U, 0xA5E50000, 2)
    rng = np.random.default_rng(0xA5)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    ob.plant_sample0(pcm, PLANTED, 0xA5)
    front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
    assert front["status"][3] == 1 and front["status"][4] == 2
    bank, T = _stretched_bank()
    return {"pcm": pcm, "front": front, "bank": bank, "T": T}


def _handle(bank, T, flags=RATE, r=0):
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    h.set_match(flags, r)
    return h


def _two_devices():
    import torch
    return torch.cuda.device_count() > 1


@pytest.mark.gpu
@pytest.mark.parametrize("r", (10, 15, 16, 118))
def test_recognise_equals_oracle_composition(case, r):
    """set_match(BAND | ANY_RATE, r): the host call on the plain and the packed transport and sr_recognise_batch_dev on a
    torch stream equal the oracle; sr_recognise_batch_multi too when two devices are visible. The guard changes the
    decision of some utterances"""
    from test_gpu_parity import _recognise_dev_np
    pcm, front, bank, T = case["pcm"], case["front"], case["bank"], case["T"]
    want = _compose(front, bank, T, RATE, r)
    band = _compose(front, bank, T, BAND, r)
    good = want["status"] == 0
    assert (want["best_idx"][good] != band["best_idx"][good]).sum() > 10, r
    h = _handle(bank, T, RATE, r)
    try:
        h.set_transport(0)
        _same(h.recognise(pcm, 2400), want, "host plain")
        h.set_transport(1)
        _same(h.recognise(pcm, 2400), want, "host packed")
        assert h.transport_stats()[0] > 0
        _same(_recognise_dev_np(h, pcm, 2400, T), want, "device launch on a torch stream")
        if _two_devices():
            h.use_own_stream()
            h2 = sr_b200.Handle(1)
            h2.set_bank(bank, T, 4096)
            h2.set_match(RATE, r)
            _same(sr_b200.recognise_multi([h, h2], pcm, 2400, want=sr_b200.RECOG_FIELDS), want, "multi")
            h2.close()
    finally:
        h.close()


@pytest.mark.gpu
def test_multi_refuses_band_beside_any_rate(case):
    """the bit is part of the matcher: sr_recognise_batch_multi over two handles (two devices when visible) refuses BAND
    beside BAND | ANY_RATE at the same radius, and runs once both carry the bit"""
    bank, T, pcm = case["bank"], case["T"], case["pcm"][:64]
    a = _handle(bank, T, RATE, 16)
    b = sr_b200.Handle(1 if _two_devices() else 0)
    b.set_bank(bank, T, 4096)
    b.set_match(BAND, 16)
    try:
        with pytest.raises(sr_b200.SrError):
            sr_b200.recognise_multi([a, b], pcm, 2400)
        b.set_match(RATE, 16)
        out = sr_b200.recognise_multi([a, b], pcm, 2400)
        assert np.array_equal(out["score"], a.recognise(pcm, 2400)["score"])
    finally:
        a.close()
        b.close()


def _check_k4(events, pool, pcm, bank, T, matcher):
    ora = ob.best_oracle()
    seg, atap = pool.segments()
    S = pcm.shape[0]
    closed = [(s, k) for s in range(S) for k in range(3) if seg[s, k, 1] != NULL]
    assert sorted((e["stream"], e["segment"]) for e, _ in events) == closed and len(closed) >= 2 * S
    for e, _ in events:
        s, k = e["stream"], e["segment"]
        f = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]), e
        if e["frm_num"] == 0:
            assert (e["status"], e["best_idx"], e["best_dis"]) == (2, 0, NULL), e
            continue
        sc = _scores(f, bank, T, *matcher)
        i = int(np.argmin(sc[0]))
        assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (0, i, int(sc[0, i]), i // 4), e


@pytest.mark.gpu
@pytest.mark.parametrize("arrival,group", [("lockstep", False), ("ragged", False), ("ragged", True)],
                         ids=["lockstep", "ragged", "group_of_two"])
def test_k4_streams_equal_oracle(case, arrival, group):
    """fixed-capture stream pushes under BAND | ANY_RATE: every event, as each push returns it, equals the oracle's
    get_mfcc of its segment, then the new oracle and the argmin; the final segment table lists exactly the events. A
    group of two handles runs on two devices only"""
    if group and not _two_devices():
        pytest.skip("a stream group across devices needs two GPUs")
    S, L = 24, 40000
    bank, T = case["bank"], case["T"]
    pcm = sr_b200.synth_pcm_host(S, L, 0xA5EDD000, 3)
    pcm[3] = 2048
    hs = [_handle(bank, T, RATE, 16)] + ([sr_b200.Handle(1)] if group else [])
    if group:
        hs[1].set_bank(bank, T, 4096)
        hs[1].set_match(RATE, 16)
    try:
        pool = sr_b200.StreamPool(hs if group else hs[0], S, L, 2400)
        events = _k4_events(pool, pcm, arrival, np.random.default_rng(0xA6))
        _check_k4(events, pool, pcm, bank, T, (RATE, 16))
        pool.close()
    finally:
        for h in hs:
            h.close()


def _synth_stretched_bank():
    """the long-recording tests' bank: 6 synthetic templates, each shrunk to every third row and stretched to three
    copies of each row (12 slots), and every third one also as it is (14 slots)"""
    tpl = sr_b200.synth_pcm_host(6, 8000, 0x7E3A0000)
    e = ob.port().recognise_batch(tpl, 2400, None, 0, 4096)
    rows = []
    for k, f in enumerate(e["ftr"]):
        x = f["mfcc_dat"][:int(f["frm_num"]) * 12].reshape(-1, 12)
        rows += [x[::3], np.repeat(x, 3, axis=0)[:119]] + ([x] if k % 3 == 0 else [])
    return sr_b200.make_bank(_ftr(rows), 4096), len(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("r", (10, 118))
def test_long_batch_and_dev_equal_oracle(r):
    """sr_recognise_long_batch and its _dev form under BAND | ANY_RATE equal the composed oracle on ragged recordings,
    and the guard changes some segments' decisions"""
    import torch
    lens = np.array([70001, 161, 123457, 99999, 200000], np.uint32)
    Ul = 200000
    pcm = ox.synth_long(len(lens), Ul, 0xA610)
    for b, n in enumerate(lens):
        pcm[b, n:] = np.where(np.arange(Ul - n) % 2, 4095, 0)
    bank, T = _synth_stretched_bank()
    h = _handle(bank, T, RATE, r)
    try:
        want = long_oracle(pcm, bank, T, RATE, r, 64, lens)
        band = long_oracle(pcm, bank, T, BAND, r, 64, lens)
        diff = sum((want["segs"][b, :int(want["n_segs"][b])]["best_idx"] != band["segs"][b, :int(band["n_segs"][b])]["best_idx"]).sum()
                   for b in range(len(lens)))
        assert diff > 0, r
        _cmp_long(h.recognise_long_batch(pcm, 64, 2400, lens), want)
        dev = torch.device("cuda:0")
        d_pcm = torch.from_numpy(pcm.view(np.int16)).to(dev)
        d_lens = torch.from_numpy(lens.view(np.int32)).to(dev)
        d_n = torch.zeros(len(lens), dtype=torch.int32, device=dev)
        d_segs = torch.zeros(len(lens) * 64 * 7, dtype=torch.int32, device=dev)
        h.recognise_long_batch_dev(d_pcm.data_ptr(), Ul, len(lens), d_lens.data_ptr(), 2400, 64, None, d_n.data_ptr(),
                                   d_segs.data_ptr())
        h.sync()
        _cmp_long(dict(n_segs=d_n.cpu().numpy().view(np.uint32),
                       segs=d_segs.cpu().numpy().view(ox.LONG_SEG_DTYPE).reshape(len(lens), 64)), want)
    finally:
        h.close()


@pytest.mark.gpu
def test_k14_long_streams_equal_oracle_on_every_prefix():
    """a live long-stream pool under BAND | ANY_RATE: each closed segment's event, handed out by the push after which it
    closed, so on the prefix pushed so far, equals the composed oracle's record of the whole recording, and every closed
    segment is handed out once"""
    xs = list(ox.synth_long(6, 120000, 0xA620))
    xs[2] = xs[2][:50000]
    bank, T = _synth_stretched_bank()
    h = _handle(bank, T, RATE, 16)
    try:
        pool = sr_b200.LongStreamPool(h, len(xs), 4000, 2400)
        events = _k14_events(pool, xs, 4000)
        pool.close()
    finally:
        h.close()
    S = len(xs)
    pcm = np.zeros((S, max(len(x) for x in xs)), np.uint16)
    lens = np.array([len(x) for x in xs], np.uint32)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    want = long_oracle(pcm, bank, T, RATE, 16, 256, lens)
    per = [0] * S
    keys = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")
    for e, _ in events:
        s, k = e["stream"], e["segment"]
        assert k == per[s]
        per[s] += 1
        rec = want["segs"][s, k]
        assert tuple(int(e[q]) for q in keys) == tuple(int(rec[q]) for q in keys), (e, rec)
    for s in range(S):
        assert per[s] == sum(1 for k in range(int(want["n_segs"][s])) if want["segs"][s, k]["status"] != 1), s
    assert sum(per) > 3 * S


# ---- launches, tags and bytes written (GPU) ----------------------------------------------------------------------------
def _tags(h):
    return [t for t, _ in h.timing_collect()]


@pytest.mark.gpu
def test_launches_and_tags_equal_the_band_matchers(case):
    """recognise, long recognise and sr_dtw_batch under BAND | ANY_RATE launch what they launch under BAND, with the
    same tags (6 for the scan), for r on both sides of every band-kernel choice"""
    pcm, bank, T = case["pcm"][:64], case["bank"], case["T"]
    lpcm = ox.synth_long(3, 100000, 0xA640)
    fin = case["front"]["ftr"][:64]
    h = _handle(bank, T, 0, 0)
    try:
        h.set_transport(0)
        h.timing_enable(4096)
        for r in (10, 15, 16, 118):
            runs = {}
            for flags in (BAND, RATE):
                h.set_match(flags, r)
                c0 = h.launch_count()
                h.recognise(pcm, 2400)
                h.recognise_long_batch(lpcm, 32, 2400)
                h.dtw(fin, flags | SIGN, r)
                runs[flags] = (h.launch_count() - c0, _tags(h))
            assert runs[RATE] == runs[BAND], r
            assert runs[RATE][1].count(DTW_BAND) == 3 and DTW not in runs[RATE][1]
    finally:
        h.close()


@pytest.mark.gpu
def test_bytes_written_equal_the_band_matchers(case):
    """sr_dtw_batch and the host recognise call under BAND | ANY_RATE write the records the band matcher writes and not
    a byte past them: every output buffer is one record longer than the call's, filled with a sentinel"""
    bank, T = case["bank"], case["T"]
    fin = case["front"]["ftr"][:40]
    B = len(fin)
    h = _handle(bank, T, RATE, 16)
    try:
        for flags in (BAND, RATE, RATE | SIGN):
            score = np.full((B + 1) * T, 0xA5A5A5A5, np.uint32)
            bi, bd = np.full(B + 1, 0xA5A5A5A5, np.uint32), np.full(B + 1, 0xA5A5A5A5, np.uint32)
            h._ck(sr_b200.lib().sr_dtw_batch(h._h, sr_b200._p(fin), B, flags, 16, sr_b200._p(score), sr_b200._p(bi),
                                              sr_b200._p(bd)))
            assert (score[B * T:] == 0xA5A5A5A5).all() and bi[B] == 0xA5A5A5A5 and bd[B] == 0xA5A5A5A5, flags
            assert (score[:B * T] != 0xA5A5A5A5).all() and (bi[:B] < T).all(), flags
        pcm = case["pcm"][:B]
        outs = {}
        for flags in (BAND, RATE):
            h.set_match(flags, 16)
            outs[flags] = h.recognise(pcm, 2400)
        for k in outs[BAND]:
            assert np.asarray(outs[RATE][k]).shape == np.asarray(outs[BAND][k]).shape, k
        _same(outs[RATE], _compose({k: v[:B] for k, v in case["front"].items()}, bank, T, RATE, 16), "recognise")
    finally:
        h.close()


# ---- real speech, reported (GPU) ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_real_speech_decisions_reported():
    """enrol each digit recording's segments (template k in slot 4k) and recognise its twin with sr_recognise_long_batch
    under band r = 118 and BAND | ANY_RATE r = 118: decisions equal the oracle; accuracy is printed, not asserted"""
    lo, port = ox.long_oracle(), ob.port()
    h = sr_b200.Handle(0)
    try:
        for a_name, b_name in _real_speech_pairs():
            a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
            bank, T, ma = _digit_bank(port, lo, a)
            h.set_bank(bank, T, 4096)
            line = []
            for flags, name in ((BAND, "band r=118"), (RATE, "band r=118 any rate")):
                h.set_match(flags, 118)
                got = h.recognise_long_batch(b[None], 32, 2400)
                _cmp_long(got, long_oracle(b[None], bank, T, flags, 118, 32))
                m = min(int(got["n_segs"][0]), ma)
                line.append("%s %d/%d" % (name, int((got["segs"][0, :m]["cmd"] == np.arange(m)).sum()), m))
            print("%s -> %s: %s" % (a_name, b_name, ", ".join(line)))
    finally:
        h.close()
