"""The bandpass lifter SR_DTW_LIFTER (an extension the reference does not have; parity unpinned) in sr_dtw_batch and on
every recognition call that reads the handle's matcher (sr_set_match).

The rule under test: with the bit, every matcher scores a pair (x, y) exactly as it scores (L(x), L(y)) without it, L
being lifter_ref.lifter on every row of the input and of the template.
CPU: the header and the binding define the bit and the weight table, and the table is round(4 (1 + 6 sin(pi k / 12)));
lifter_ref.lifter saturates at the s16 edges and nowhere else; the composed oracle (lifter_ref.match_scores) equals the
plain band and any-rate DPs of refs.py on liftered rows, and reproduces the real-speech figures of the four digit recordings.
GPU: the setter's flag rules; sr_dtw_batch with the bit equals sr_dtw_batch without it on pre-liftered inputs and bank,
under all four matchers at radii that pick each band kernel, on every (I, M) in 1..119 x 1..119, with rows that saturate;
every recognition path (host plain and packed, _dev, _multi, the long-form host and _dev calls, fixed-capture pools and
live long streams) under each matcher with the bit, and with the decision rules on top, equals the oracle composition;
_multi refuses a lifter/plain mix; launches, timing tags and bytes written are the flag-off matcher's.
sr_recognise_batch_dev_allgather is run on a one-rank communicator by test_decision_paths.py; stream groups over two
devices are not run here: they need two GPUs.
Every GPU test makes its own handles."""
import os
import re

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import bank_planted, digit_bank, inputs, make_ftr, real_speech_pairs, synth_long_poisoned, tie_rows
from drive import LONG_REC, cmp_long, handle, k4_events, k14_events, recognise_dev_np, recognise_long_dev_np, same, tags
from lifter_ref import compose_recognise, lifter, lifter_bank, lifter_ftr, match_scores, recognise_long
from refs import band_dp_ref, rate_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIS_ERR = 0xFFFFFFFF
BAND, SIGN, SYM, ANY, LIFT = sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN, sr_b200.DTW_SYM_P1, sr_b200.DTW_ANY_RATE, sr_b200.DTW_LIFTER
RATE = BAND | ANY
KNN, REJ = sr_b200.dtw_knn, sr_b200.dtw_reject
W = (10, 16, 21, 25, 27, 28, 27, 25, 21, 16, 10, 4)
# (flags, r) of the recognition matchers: the greedy walk, the band DP's three kernels, any-rate, the symmetric DP
MATCHERS = ((0, 0), (BAND, 5), (BAND, 10), (BAND, 16), (RATE, 118), (SYM, 10))
# radii of sr_dtw_batch: the warp-scan band kernel (0, 15), the thread form (10), the whole-row kernel (16, 118)
KERNEL_RADII = (0, 10, 15, 16, 118)
# tags of sr_timing_collect
DTW, DTW_BAND, DTW_SYM = 4, 6, 14


def _ids(m):
    return "%d_r%d" % m


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_header_and_binding_define_the_bit_and_table():
    with open(os.path.join(ROOT, "include", "speech_recog.h")) as f:
        hdr = f.read()
    m = re.search(r"#define\s+SR_DTW_LIFTER\s+\(1u\s*<<\s*(\d+)\)", hdr)
    assert m and int(m.group(1)) == 13
    m = re.search(r"#define\s+SR_DTW_LIFTER_W\s+\{([^}]*)\}", hdr)
    assert m and tuple(int(v) for v in m.group(1).split(",")) == W
    assert sr_b200.DTW_LIFTER == 1 << 13 and tuple(sr_b200.DTW_LIFTER_W) == W
    k = np.arange(1, 13)
    assert tuple(int(v) for v in np.round(4 * (1 + 6 * np.sin(np.pi * k / 12)))) == W
    taken = BAND | SIGN | SYM | ANY | (7 << 8) | REJ(0xFFFF)
    assert LIFT & taken == 0


def test_lifter_saturates_at_the_s16_edges():
    """lifter_ref.lifter on every s16 value in every coefficient equals sat16(trunc(a * W / 16)) in Python integers; it
    saturates exactly where |a| * W / 16 leaves the s16 range (first at |a| = 18 725 for W = 28) and keeps every value
    within 1.75x of the original"""
    a = np.arange(-32768, 32768, dtype=np.int64)
    rows = np.repeat(a[:, None], 12, axis=1).astype(np.int16)
    got = lifter(rows).astype(np.int64)
    for c, w in enumerate(W):
        p = a * w
        want = np.clip(np.where(p < 0, -((-p) // 16), p // 16), -32768, 32767)
        assert np.array_equal(got[:, c], want), c
        sat = (p >= 32768 * 16) | (p <= -32769 * 16)                      # trunc(p / 16) outside [-32768, 32767]
        assert np.array_equal(np.flatnonzero(sat), np.flatnonzero(np.abs(a) * w >= 32768 * 16 + (a < 0) * 16)), c
        assert (np.abs(a[sat]) >= 18725).all(), c
    assert (np.abs(got) <= np.ceil(1.75 * np.abs(a))[:, None]).all()
    assert (got[a == 32767] == [20479, 32767, 32767, 32767, 32767, 32767, 32767, 32767, 32767, 32767, 20479, 8191]).all()
    assert (got[a == -32768] == [-20480] + [-32768] * 9 + [-20480, -8192]).all()
    small = np.abs(a) <= 18724
    assert (np.abs(got[small]) < 32768).all() and got[a == 18724][0, 5] == 32767
    assert got[a == 18725][0, 5] == 32767 and got[a == -18725][0, 5] == -32768   # the first saturated values
    assert got[a == -1][0].tolist() == [0, -1, -1, -1, -1, -1, -1, -1, -1, -1, 0, 0]  # truncation toward zero
    assert lifter(rows[:24].reshape(2, 144)).tolist() == got[:24].reshape(2, 144).tolist()


def test_composed_oracle_equals_plain_dps_on_liftered_rows():
    """match_scores under BAND | LIFTER and BAND | ANY_RATE | LIFTER equals refs.band_dp_ref and refs.rate_ref on the
    liftered rows, on pairs with saturating rows and across the 2:1 guard; the bank's headers and unused bytes stay"""
    rng = np.random.default_rng(0x11F)
    frms = [1, 2, 5, 9, 14, 20]
    xs = [tie_rows(rng, f, ("small", "full", "tie")[k % 3]) for k, f in enumerate(frms)]
    ys = [tie_rows(rng, f, ("full", "small", "tie")[k % 3]) for k, f in enumerate(frms[::-1])]
    fin = make_ftr(xs)
    bank = sr_b200.make_bank(make_ftr(ys), 4096)
    lb = lifter_bank(bank, len(ys))
    assert lb.shape == bank.shape and np.array_equal(lb[:, :4], bank[:, :4])
    assert np.array_equal(lb[:, ob.FTR_DTYPE.itemsize:], bank[:, ob.FTR_DTYPE.itemsize:])
    for r in (0, 3, 118):
        band = match_scores(fin, bank, len(ys), BAND | LIFT, r)
        rate = match_scores(fin, bank, len(ys), RATE | LIFT, r)
        for i, x in enumerate(xs):
            for j, y in enumerate(ys):
                assert band[i, j] == band_dp_ref(lifter(x), lifter(y), r), (r, i, j)
                d = rate_ref(lifter(x), lifter(y), r)
                assert rate[i, j] == (DIS_ERR if d is None else d // (len(x) + len(y))), (r, i, j)
    assert (match_scores(fin, bank, len(ys), BAND | LIFT, 118) != match_scores(fin, bank, len(ys), BAND, 118)).any()


def test_real_speech_accuracy_on_the_oracles():
    """the digit recordings, each recognised against its twin's segments at r = 118, plain and liftered: words right per
    recording. A fixed computation on fixed data, not a claim about speech in general"""
    lo, port = ox.long_oracle(), ob.port()
    got = {}
    for a_name, b_name in real_speech_pairs():
        a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
        bank, T, ma = digit_bank(port, lo, a)
        for flags in (BAND, RATE, SYM, 0):
            for lift in (0, LIFT):
                w = recognise_long(lo, port, b[None], 2400, bank, T, 4096, 32, match=(flags | lift, 118))
                m = min(int(w["n_segs"][0]), ma)
                got.setdefault((flags, lift), []).append(int((w["segs"][0, :m]["cmd"] == np.arange(m)).sum()))
    assert got == {(BAND, 0): [6, 8, 3, 3], (BAND, LIFT): [5, 8, 3, 3],
                   (RATE, 0): [4, 8, 9, 8], (RATE, LIFT): [4, 8, 10, 10],
                   (SYM, 0): [6, 7, 3, 2], (SYM, LIFT): [6, 7, 3, 1],
                   (0, 0): [6, 7, 3, 3], (0, LIFT): [6, 7, 3, 3]}, got


# ---- the setter (GPU) --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_match_rules_with_the_lifter():
    """LIFTER with every matcher, KNN(0..4) and REJ(q) round-trips through sr_get_match; a value refused without the bit
    is refused with it, and a refused call leaves the setting unchanged"""
    h = sr_b200.Handle(0)
    try:
        for flags, r in MATCHERS:
            for k in (0, 1, 4):
                for q in (0, 100, 65535):
                    h.set_match(flags | LIFT | KNN(k) | REJ(q), r)
                    assert h.match() == (flags | LIFT | KNN(k) | REJ(q), r)
        h.set_match(SYM | LIFT | KNN(2) | REJ(9), 7)
        bad = [(LIFT | ANY, 3), (LIFT | SYM | BAND, 3), (LIFT | SYM | ANY, 3), (LIFT | SIGN, 3), (LIFT | BAND, -1),
               (LIFT | (5 << 8), 3), (LIFT | (7 << 8) | BAND, 3)]
        bad += [(LIFT | flags | (1 << b), r) for flags, r in MATCHERS[:2] for b in (4, 5, 6, 7, 11, 12, 14, 15)]
        for flags, r in bad:
            with pytest.raises(sr_b200.SrError):
                h.set_match(flags, r)
            assert h.match() == (SYM | LIFT | KNN(2) | REJ(9), 7), hex(flags)
    finally:
        h.close()


# ---- sr_dtw_batch: the metamorphic rule (GPU) -----------------------------------------------------------------------------
def _every_shape_case(kind, seed):
    """inputs of 1..119 frames against a 119-slot bank of 119..1 frames: every (I, M) in 1..119 x 1..119 once. "full" rows
    are +-32 767, so every coefficient but the first, the eleventh and the twelfth saturates"""
    rng = np.random.default_rng(seed)
    frms = list(range(1, 120))
    fin = make_ftr([tie_rows(rng, f, kind) for f in frms])
    bank = sr_b200.make_bank(make_ftr([tie_rows(rng, f, kind) for f in frms[::-1]]), 4096)
    return fin, bank


def _scan_matchers():
    """(flags, r, greedy kernel variant) of every scan kernel: both greedy forms, the band DP and any-rate at each band
    kernel's radii, the symmetric DP"""
    out = [(0, 0, 0), (0, 0, 1)]
    out += [(f, r, 0) for f in (BAND, RATE) for r in KERNEL_RADII]
    out += [(SYM, r, 0) for r in (0, 10, 16, 118)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("small", "full"))
def test_dtw_batch_liftered_equals_plain_on_liftered_rows(kind):
    """score, best_idx and best_dis of sr_dtw_batch(flags | LIFTER) on every (I, M) in 1..119 x 1..119 equal
    sr_dtw_batch(flags) on the liftered inputs against the liftered bank, bit for bit, under every scan kernel; the
    liftered scores differ from the plain ones"""
    fin, bank = _every_shape_case(kind, 0x11F0 + (kind == "full"))
    lfin, lbank = lifter_ftr(fin), lifter_bank(bank, 119)
    if kind == "full":
        assert (np.abs(lfin["mfcc_dat"][:, 12:]) == 32767).any()          # saturated rows
    h, hl = sr_b200.Handle(0), sr_b200.Handle(0)
    h.set_bank(bank, 119, 4096)
    hl.set_bank(lbank, 119, 4096)
    try:
        for flags, r, v in _scan_matchers():
            h.set_dtw_variant(v)
            hl.set_dtw_variant(v)
            got = h.dtw(fin, flags=flags | LIFT, band_r=r)
            want = hl.dtw(lfin, flags=flags, band_r=r)
            for g, w, what in zip(got, want, ("score", "best_idx", "best_dis")):
                assert np.array_equal(g, w), (kind, flags, r, v, what, np.argwhere(g != w)[:4].tolist())
            assert (got[0] != h.dtw(fin, flags=flags, band_r=r)[0]).any(), (kind, flags, r, v)
    finally:
        h.close()
        hl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", (1, 33, 80))
def test_dtw_batch_planted_slots_liftered_equal_plain(T):
    """banks with erased, unsigned, frm_num 0 and frm_num 120 slots; inputs of 0..120 frames: with and without
    CHECK_SIGN, the bit equals the liftered inputs and bank without it, and under CHECK_SIGN equals the composed oracle
    on the pairs it is defined for (frm_num <= 119 on both sides)"""
    rng = np.random.default_rng(0x11F4 + T)
    bank = bank_planted(rng, T)
    frms = [0, 120, 1, 119, 2, 118, 3, 100] + [int(x) for x in rng.integers(1, 120, 32)]
    fin = inputs(rng, frms)
    lfin, lbank = lifter_ftr(fin), lifter_bank(bank, T)
    h, hl = sr_b200.Handle(0), sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    hl.set_bank(lbank, T, 4096)
    try:
        for flags, r, v in _scan_matchers():
            h.set_dtw_variant(v)
            hl.set_dtw_variant(v)
            for sign in (0, SIGN):
                got = h.dtw(fin, flags=flags | sign | LIFT, band_r=r)
                want = hl.dtw(lfin, flags=flags | sign, band_r=r)
                for g, w in zip(got, want):
                    assert np.array_equal(g, w), (T, flags, r, v, sign)
            if v == 0:                                       # the oracles where both sides have at most 119 frames
                keep = fin["frm_num"] <= 119
                cols = (bank[:, 2].astype(int) | bank[:, 3].astype(int) << 8) <= 119
                want = match_scores(fin[keep], bank, T, flags | LIFT, r)
                assert np.array_equal(got[0][keep][:, cols], want[:, cols]), (T, flags, r)
    finally:
        h.close()
        hl.close()


# ---- recognition under the lifter (GPU) ------------------------------------------------------------------------------------
U = 16000


@pytest.fixture(scope="module")
def case():
    """3 200 two-second utterances (the packed transport engages), a silent one, one over 119 frames; 12 synthetic
    templates, one of them unsigned"""
    B = 3200
    pcm = sr_b200.synth_pcm_host(B, U, 0x11F50000, 2)
    rng = np.random.default_rng(0x11F5)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
    assert front["status"][3] == 1 and front["status"][4] == 2
    tpl = sr_b200.synth_pcm_host(12, 8000, 0x7E3A0000)
    e = ob.port().recognise_batch(tpl, 2400, None, 0, 4096)
    valid = np.ones(12, bool)
    valid[5] = False
    return {"pcm": pcm, "front": front, "bank": sr_b200.make_bank(e["ftr"], 4096, valid), "T": 12}


def _two_devices():
    import torch
    return torch.cuda.device_count() > 1


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", MATCHERS, ids=_ids)
def test_recognise_equals_oracle_composition(case, matcher):
    """set_match(flags | LIFTER, r): the host call on the plain and the packed transport and sr_recognise_batch_dev on a
    torch stream equal the oracle composition, then under KNN(3) | REJ(100) the numpy rule on its scores;
    sr_recognise_batch_multi too when two devices are visible. The lifter changes scores"""
    flags, r = matcher
    pcm, front, bank, T = case["pcm"], case["front"], case["bank"], case["T"]
    want = compose_recognise(front, bank, T, flags | LIFT, r)
    plain = compose_recognise(front, bank, T, flags, r)
    assert (want["score"] != plain["score"]).any()
    h = handle(bank, T, flags | LIFT, r)
    try:
        h.set_transport(0)
        same(h.recognise(pcm, 2400), want, "host plain")
        h.set_transport(1)
        same(h.recognise(pcm, 2400), want, "host packed")
        assert h.transport_stats()[0] > 0
        same(recognise_dev_np(h, pcm, 2400, T), want, "device launch on a torch stream")
        h.use_own_stream()
        h.set_match(flags | LIFT | KNN(3) | REJ(100), r)
        h.set_transport(0)
        same(h.recognise(pcm[:400], 2400), ox.under_rule({k: v[:400] for k, v in want.items()}, 3, 100), "rules")
        if _two_devices():
            h.set_match(flags | LIFT, r)
            h2 = sr_b200.Handle(1)
            h2.set_bank(bank, T, 4096)
            h2.set_match(flags | LIFT, r)
            same(sr_b200.recognise_multi([h, h2], pcm, 2400, want=sr_b200.RECOG_FIELDS), want, "multi")
            h2.close()
    finally:
        h.close()


@pytest.mark.gpu
def test_multi_refuses_a_lifter_plain_mix(case):
    """the bit is part of the matcher: sr_recognise_batch_multi over two handles (two devices when visible) refuses a
    liftered handle beside a plain one of the same matcher, with no launch, and runs once both carry the bit"""
    bank, T, pcm = case["bank"], case["T"], case["pcm"][:64]
    a = handle(bank, T, BAND | LIFT, 16)
    b = sr_b200.Handle(1 if _two_devices() else 0)
    b.set_bank(bank, T, 4096)
    try:
        for other, r in ((BAND, 16), (0, 0), (LIFT, 0), (BAND | LIFT, 10)):
            b.set_match(other, r)
            ca, cb = a.launch_count(), b.launch_count()
            with pytest.raises(sr_b200.SrError):
                sr_b200.recognise_multi([a, b], pcm, 2400)
            assert (a.launch_count(), b.launch_count()) == (ca, cb)
        b.set_match(BAND | LIFT, 16)
        out = sr_b200.recognise_multi([a, b], pcm, 2400)
        assert np.array_equal(out["score"], a.recognise(pcm, 2400)["score"])
    finally:
        a.close()
        b.close()


def _check_k4(events, pool, pcm, bank, T, matcher):
    """every closed segment has one event, and each equals the oracle's get_mfcc of its segment, then the scan under the
    matcher and the first-wins argmin"""
    ora = ob.best_oracle()
    seg, atap = pool.segments()
    S = pcm.shape[0]
    closed = [(s, k) for s in range(S) for k in range(3) if seg[s, k, 1] != DIS_ERR]
    assert sorted((e["stream"], e["segment"]) for e, _ in events) == closed and len(closed) >= 2 * S
    for e, _ in events:
        s, k = e["stream"], e["segment"]
        f = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]), e
        if e["frm_num"] == 0:
            assert (e["status"], e["best_idx"], e["best_dis"]) == (2, 0, DIS_ERR), e
            continue
        sc = match_scores(f, bank, T, *matcher)
        i = int(np.argmin(sc[0]))
        assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (0, i, int(sc[0, i]), i // 4), e


def _check_k14(events, xs, bank, T, matcher):
    """each event equals the composed oracle's record of its whole recording, in segment order, and every closed segment
    is handed out once"""
    S, Ul = len(xs), max(len(x) for x in xs)
    pcm = np.zeros((S, Ul), np.uint16)
    lens = np.array([len(x) for x in xs], np.uint32)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    w = recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, T, 4096, 256, lens, match=matcher)
    per = [0] * S
    for e, _ in events:
        s, k = e["stream"], e["segment"]
        assert k == per[s], (s, k, per[s])
        per[s] += 1
        rec = w["segs"][s, k]
        assert tuple(int(e[q]) for q in LONG_REC) == tuple(int(rec[q]) for q in LONG_REC), (e, rec)
    for s in range(S):
        assert per[s] == sum(1 for k in range(int(w["n_segs"][s])) if w["segs"][s, k]["status"] != 1), s
    assert sum(per) > 3 * S, per


@pytest.mark.gpu
def test_k4_streams_equal_oracle(case):
    """fixed-capture stream pushes under BAND | LIFTER: every event equals the oracle's get_mfcc of its segment, the
    liftered scan and the argmin; the final segment table lists exactly the events"""
    S, L = 24, 40000
    bank, T = case["bank"], case["T"]
    pcm = sr_b200.synth_pcm_host(S, L, 0x11F6D000, 3)
    pcm[3] = 2048
    h = handle(bank, T, BAND | LIFT, 16)
    try:
        pool = sr_b200.StreamPool(h, S, L, 2400)
        events = k4_events(pool, pcm, "ragged", np.random.default_rng(0x11F6))
        _check_k4(events, pool, pcm, bank, T, (BAND | LIFT, 16))
        pool.close()
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", ((0, 0), (RATE, 118), (SYM, 10)), ids=_ids)
def test_long_batch_and_dev_equal_oracle(matcher):
    """sr_recognise_long_batch and its _dev form under flags | LIFTER equal the composed oracle on ragged recordings"""
    flags, r = matcher
    lens = np.array([70001, 161, 123457, 99999, 200000], np.uint32)
    pcm = synth_long_poisoned(lens, 200000, 0x11F7)
    bank, T = ox.synth_bank(12)
    h = handle(bank, T, flags | LIFT, r)
    try:
        want = recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, T, 4096, 64, lens, match=(flags | LIFT, r))
        cmp_long(h.recognise_long_batch(pcm, 64, 2400, lens), want)
        cmp_long(recognise_long_dev_np(h, pcm, lens, 64), want)
    finally:
        h.close()


@pytest.mark.gpu
def test_k14_long_streams_equal_oracle_on_every_prefix():
    """a live long-stream pool under SYM_P1 | LIFTER: each closed segment's event, handed out by the push after which it
    closed, equals the composed oracle's record of the whole recording, and every closed segment is handed out once"""
    xs = list(ox.synth_long(6, 120000, 0x11F8))
    xs[2] = xs[2][:50000]
    bank, T = ox.synth_bank(12)
    h = handle(bank, T, SYM | LIFT, 10)
    try:
        pool = sr_b200.LongStreamPool(h, len(xs), 4000, 2400)
        events = k14_events(pool, xs, 4000)
        pool.close()
    finally:
        h.close()
    _check_k14(events, xs, bank, T, (SYM | LIFT, 10))


# ---- launches, tags and bytes written (GPU) ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_launches_and_tags_equal_the_flag_off_matchers(case):
    """recognise, long recognise and sr_dtw_batch under flags | LIFTER launch what they launch under flags, with the
    same tags (4, 6 or 14 for the scan), for every matcher"""
    pcm, bank, T = case["pcm"][:64], case["bank"], case["T"]
    lpcm = ox.synth_long(3, 100000, 0x11F9)
    fin = case["front"]["ftr"][:64]
    h = handle(bank, T, 0, 0)
    try:
        h.set_transport(0)
        h.timing_enable(4096)
        for flags, r in MATCHERS:
            runs = {}
            for lift in (0, LIFT):
                h.set_match(flags | lift, r)
                c0 = h.launch_count()
                h.recognise(pcm, 2400)
                h.recognise_long_batch(lpcm, 32, 2400)
                h.dtw(fin, flags | lift | SIGN, r)
                runs[lift] = (h.launch_count() - c0, tags(h))
            assert runs[LIFT] == runs[0], (flags, r)
            scan = DTW_SYM if flags & SYM else DTW_BAND if flags & BAND else DTW
            assert runs[LIFT][1].count(scan) == 3, (flags, r)
    finally:
        h.close()


@pytest.mark.gpu
def test_bytes_written_equal_the_flag_off_matchers(case):
    """sr_dtw_batch and the host recognise call under flags | LIFTER write the records the flag-off matcher writes and not
    a byte past them: every output buffer is one record longer than the call's, filled with a sentinel"""
    bank, T = case["bank"], case["T"]
    fin = case["front"]["ftr"][:40]
    B = len(fin)
    pcm = case["pcm"][:B]
    h = handle(bank, T, 0, 0)
    try:
        for flags, r in MATCHERS:
            outs = {}
            for lift in (0, LIFT):
                score = np.full((B + 1) * T, 0xA5A5A5A5, np.uint32)
                bi, bd = np.full(B + 1, 0xA5A5A5A5, np.uint32), np.full(B + 1, 0xA5A5A5A5, np.uint32)
                h._ck(sr_b200.lib().sr_dtw_batch(h._h, sr_b200._p(fin), B, flags | lift, r, sr_b200._p(score),
                                                  sr_b200._p(bi), sr_b200._p(bd)))
                assert (score[B * T:] == 0xA5A5A5A5).all() and bi[B] == 0xA5A5A5A5 and bd[B] == 0xA5A5A5A5, (flags, lift)
                assert (score[:B * T] != 0xA5A5A5A5).all() and (bi[:B] < T).all(), (flags, lift)
                h.set_match(flags | lift, r)
                outs[lift] = h.recognise(pcm, 2400)
            for k in outs[0]:
                assert np.asarray(outs[LIFT][k]).shape == np.asarray(outs[0][k]).shape, k
            want = compose_recognise({k: v[:B] for k, v in case["front"].items()}, bank, T, flags | LIFT, r)
            same(outs[LIFT], want, ("recognise", flags, r))
    finally:
        h.close()
