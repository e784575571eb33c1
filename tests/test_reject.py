"""The runner-up margin rule SR_DTW_REJECT(q) (an extension: the reference always names a command) on every recognition
call that reads the handle's matcher.

CPU: the header and the binding define the rule, its status and ABI version 12; a vectorised reference of the rule equals a
brute force over random score rows; the real-speech table of DESIGN.md is recomputed from the oracles. GPU: the setter and
flag rules; sr_dtw_batch* refuse the rule's bits before anything runs; every recognition path under each matcher at several
q equals the same call without the rule except for SR_ST_REJECT, which appears exactly where the rule, applied to the
oracle-checked scores, says; banks of 1 .. 1024 slots and batches around the grid's row count; launches, timing tags and
bytes written are the rule-off call's; unequal rules are refused by _multi and groups; two threads with different rules.
sr_recognise_batch_dev_allgather is run on a one-rank communicator by test_decision_paths.py."""
import os
import re
import threading

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import bank_planted, digit_bank, inputs, real_speech_pairs, synth_long_poisoned
from drive import event_key, handle, k4_events, k14_events, recognise_dev_np, recognise_long_dev_np
from refs import decide

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = DIS_ERR = 0xFFFFFFFF
BAND, SIGN, SYM, ANY = sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN, sr_b200.DTW_SYM_P1, sr_b200.DTW_ANY_RATE
RATE = BAND | ANY
REJ = sr_b200.dtw_reject
OK, REJECT = sr_b200.ST_OK, sr_b200.ST_REJECT
# (flags, r): the greedy walk, the three band kernels (warp-scan r = 5, thread form r = 10, whole row r = 16), any-rate at
# the full matrix, the symmetric DP
MATCHERS = ((0, 0), (BAND, 5), (BAND, 10), (BAND, 16), (RATE, 118), (SYM, 10))
QS = (1, 100, 1000, 65535)


# ---- the rule in Python --------------------------------------------------------------------------------------------------
def rule_brute(row, q):
    """the rule on one score row with Python integers: the winner, then every other command's best score"""
    T = len(row)
    c1 = min(range(T), key=lambda t: (int(row[t]), t)) // 4
    d1 = min(int(v) for v in row)
    runners = [int(row[t]) for t in range(T) if t // 4 != c1]
    if not runners or min(runners) == DIS_ERR:
        return False
    return 1000 * (min(runners) - d1) < q * d1


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_header_and_binding_define_the_rule():
    with open(os.path.join(ROOT, "include", "speech_recog.h")) as f:
        text = f.read()
    m = re.search(r"#define\s+SR_DTW_REJECT\(q\)\s+\(\(uint32_t\)\(q\)\s*<<\s*16\)", text)
    assert m, "SR_DTW_REJECT"
    m = re.search(r"#define\s+SR_ST_REJECT\s+(\w+)", text)
    assert m and int(m.group(1).rstrip("uU"), 0) == 3
    assert sr_b200.ST_REJECT == 3 and sr_b200.dtw_reject(1) == 1 << 16 and sr_b200.dtw_reject(65535) == 0xFFFF0000
    assert sr_b200.dtw_reject(0) == 0
    for bad in (-1, 65536):
        with pytest.raises(ValueError):
            sr_b200.dtw_reject(bad)
    assert sr_b200.lib().sr_abi_version() == 12


def test_rule_reference_equals_brute_force():
    """refs.decide(score, 1, q) == rule_brute on random rows: ties between commands, d1 = 0, all-SR_DIS_ERR runner-ups,
    T not a multiple of 4, one-command banks, q = 1 and q = 65535"""
    rng = np.random.default_rng(0x7E1)
    seen = dict(tie=0, zero=0, err_runner=0, one_cmd=0, rej=0, keep=0)
    for T in (1, 2, 3, 4, 5, 7, 8, 9, 13, 33, 80):
        for q in (1, 2, 100, 999, 1000, 65535):
            for kind in ("wide", "tight", "tie", "zero", "err"):
                B = 64
                if kind == "wide":
                    sc = rng.integers(0, 65536, (B, T))
                elif kind == "tight":
                    sc = 1000 + rng.integers(0, 3, (B, T))
                elif kind == "tie":
                    sc = np.full((B, T), 700) + rng.integers(0, 2, (B, T)) * (rng.integers(0, 2, (B, 1)))
                elif kind == "zero":
                    sc = rng.integers(0, 3, (B, T))
                else:
                    sc = rng.integers(1, 5000, (B, T))
                    sc[rng.random((B, T)) < 0.6] = DIS_ERR
                sc = sc.astype(np.uint32)
                _, d1, _, rej = decide(sc, 1, q)
                for b in range(B):
                    assert bool(rej[b]) == rule_brute(sc[b], q), (T, q, kind, sc[b].tolist())
                seen["one_cmd"] += T <= 4
                seen["zero"] += int((d1 == 0).sum())
                seen["rej"] += int(rej.sum())
                seen["keep"] += int((~rej).sum())
                if kind == "tie" and T > 4:
                    seen["tie"] += 1
                if kind == "err" and T > 4:
                    seen["err_runner"] += 1
    assert all(v > 0 for v in seen.values()), seen


def _margin_table(q):
    """per digit-recording pair: the first half of one recording's words enrolled (one template per command), every word
    of its twin recognised at r = 118 without the 2:1 guard, then the rule at q. (in-vocabulary words, kept, kept and
    right, out-of-vocabulary words, rejected)"""
    lo, port = ox.long_oracle(), ob.port()
    rows = []
    for a_name, b_name in real_speech_pairs():
        a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
        bank, T, ma = digit_bank(port, lo, a)
        half = ma // 2
        bank = bank.copy()
        bank[4 * half:, 0:2] = 0xFF                                  # words half .. ma - 1 not enrolled: unsigned slots
        w = ox.recognise_long(lo, port, b[None], 2400, bank, T, 4096, 32, match=(RATE, 118))
        m = min(int(w["n_segs"][0]), ma)
        segs = w["segs"][0, :m]
        todo = [k for k in range(m) if segs[k]["status"] == OK]
        ftr = ox.ftr_of_segments(port, b[None], w["atap"], [(0, int(segs[k]["start"]), int(segs[k]["end"])) for k in todo])
        sc = ox.match_scores(ftr, bank, T, RATE, 118)
        idx, _, _, rej = decide(sc, 1, q)
        inv = np.array([k < half for k in todo])
        right = idx // 4 == np.array(todo)
        rows.append((int(inv.sum()), int((inv & ~rej).sum()), int((inv & ~rej & right).sum()), int((~inv).sum()),
                     int((~inv & rej).sum())))
    return rows


def test_real_speech_margin_table():
    """the table of DESIGN.md: a fixed computation on the four digit recordings, not a claim about speech in general"""
    assert _margin_table(100) == REAL_SPEECH_Q100, _margin_table(100)
    assert _margin_table(0) == REAL_SPEECH_Q0, _margin_table(0)


# (in-vocabulary words, kept, kept and right, out-of-vocabulary words, rejected) per pair; without the rule every word is
# kept and 17 of the 22 in-vocabulary words are right, at q = 100 16 are kept (15 right) and 14 of the 24 others rejected
REAL_SPEECH_Q0 = [(5, 5, 3, 5, 0), (5, 5, 4, 5, 0), (6, 6, 5, 7, 0), (6, 6, 5, 7, 0)]
REAL_SPEECH_Q100 = [(5, 2, 2, 5, 3), (5, 5, 4, 5, 0), (6, 5, 5, 7, 7), (6, 4, 4, 7, 4)]


# ---- GPU: setter and flag rules ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_match_rules_with_the_rule():
    """every matcher | REJECT(q) round-trips through sr_get_match; what the setter refused before it still refuses with
    the rule's bits, and a refused call leaves the setting unchanged"""
    h = sr_b200.Handle(0)
    try:
        for flags, r in MATCHERS:
            for q in (0,) + QS:
                h.set_match(flags | REJ(q), r)
                assert h.match() == (flags | REJ(q), r)
        h.set_match(BAND | REJ(77), 7)
        for flags, r in ((ANY | REJ(5), 3), (SYM | BAND | REJ(5), 3), (ANY | SYM | REJ(5), 3), (SIGN | REJ(5), 3),
                         (BAND | REJ(5), -1), (16 | REJ(5), 3), (0x8000 | REJ(5), 3)):
            with pytest.raises(sr_b200.SrError):
                h.set_match(flags, r)
            assert h.match() == (BAND | REJ(77), 7)
    finally:
        h.close()


@pytest.mark.gpu
def test_dtw_batch_refuses_the_rule_bits():
    """sr_dtw_batch and sr_dtw_batch_dev have no status to report a rejection in: any bit >= 16 fails with no launch and
    no output byte written, under every matcher"""
    import torch
    h = sr_b200.Handle(0)
    try:
        rng = np.random.default_rng(0x7E2)
        h.set_bank(bank_planted(rng, 8), 8, 4096)
        fin = inputs(rng, [30, 40, 50])
        score = np.full((3, 8), 0xA5A5A5A5, np.uint32)
        bi, bd = np.full(3, 0xA5A5A5A5, np.uint32), np.full(3, 0xA5A5A5A5, np.uint32)
        dev = torch.device("cuda:0")
        d_in = torch.from_numpy(fin.view(np.uint8).copy()).to(dev)
        d_out = [torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device=dev) for n in (24, 3, 3)]
        c0 = h.launch_count()
        for flags, r in MATCHERS:
            for bits in (REJ(1), REJ(100), REJ(65535), 1 << 16, 1 << 31):
                with pytest.raises(sr_b200.SrError):
                    h._ck(sr_b200.lib().sr_dtw_batch(h._h, sr_b200._p(fin), 3, flags | SIGN | bits, r, sr_b200._p(score),
                                                      sr_b200._p(bi), sr_b200._p(bd)))
                with pytest.raises(sr_b200.SrError):
                    h.dtw_dev(d_in.data_ptr(), 3, flags | bits, r, *[t.data_ptr() for t in d_out])
        h.sync()
        assert h.launch_count() == c0
        assert (score == 0xA5A5A5A5).all() and (bi == 0xA5A5A5A5).all() and (bd == 0xA5A5A5A5).all()
        assert all((t == 0x5A5A5A5A).all().item() for t in d_out)
    finally:
        h.close()


# ---- GPU: recognition under the rule ------------------------------------------------------------------------------------
U = 16000


def _bank_of(n_slot, seed):
    """n_slot signed templates from synthetic utterances: commands of four near-identical slots (the same words with
    one row dropped), so that a command's own second slot is always closer than another command"""
    n_cmd = (n_slot + 3) // 4
    tpl = sr_b200.synth_pcm_host(n_cmd, 8000, seed)
    e = ob.recognise_pinned(ob.best_oracle(), tpl, 2400, None, 0, 4096)
    ftr = np.zeros(4 * n_cmd, ob.FTR_DTYPE)
    for c in range(n_cmd):
        f = e["ftr"][c] if e["status"][c] == OK else e["ftr"][0]
        n = int(f["frm_num"])
        rows = f["mfcc_dat"][:n * 12].reshape(n, 12)
        for k in range(4):
            x = rows if k == 0 else np.delete(rows, min(k * 7, n - 1), axis=0)
            ftr[4 * c + k]["frm_num"] = len(x)
            ftr[4 * c + k]["mfcc_dat"][:x.size] = x.reshape(-1)
    return sr_b200.make_bank(ftr[:n_slot], 4096)


@pytest.fixture(scope="module")
def case():
    """700 two-second synthetic utterances with a silent one and one over 119 frames; an 80-slot bank"""
    B = 700
    pcm = sr_b200.synth_pcm_host(B, U, 0x7E350000, 2)
    rng = np.random.default_rng(0x7E3)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
    assert front["status"][3] == 1 and front["status"][4] == 2
    return {"pcm": pcm, "front": front, "bank": _bank_of(80, 0x7E3A0000), "T": 80}


def _same_but_status(on, off, q, what):
    """the rule-on result equals the rule-off one field by field, except status, which is the rule on off's scores"""
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd"):
        assert np.array_equal(np.asarray(on[k]), np.asarray(off[k])), (what, q, k)
    assert ob.ftr_equal(on["ftr"], off["ftr"]), what
    want = ox.under_rule(off, 1, q)["status"]
    bad = np.flatnonzero(np.asarray(on["status"]) != want)
    assert len(bad) == 0, (what, q, bad[:8].tolist())
    return int((want == REJECT).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", MATCHERS, ids=lambda m: "%d_r%d" % m)
def test_recognise_paths_equal_oracle_and_rule(case, matcher):
    """under each matcher: the rule-off host call equals the oracle composition; then, at every q, the host call on the
    plain and the packed transport and sr_recognise_batch_dev on a torch stream equal it except for SR_ST_REJECT, which
    is exactly the rule on the oracle's scores; launch counts and timing tags are the rule-off call's. Rejections grow
    with q, and q = 100 keeps some decisions"""
    flags, r = matcher
    pcm, front, bank, T = case["pcm"], case["front"], case["bank"], case["T"]
    good = front["status"] == OK
    sc = ox.match_scores(front["ftr"][good], bank, T, flags, r)
    h = handle(bank, T, flags, r)
    try:
        h.set_transport(0)
        h.timing_enable(64)
        off = h.recognise(pcm, 2400)
        assert np.array_equal(off["score"][good], sc) and (off["status"] == front["status"]).all()
        tags_off = [t for t, _ in h.timing_collect()]
        dev_off = recognise_dev_np(h, pcm, 2400, T)
        h.use_own_stream()
        h.timing_collect()
        n_rej = {}
        for q in QS:
            h.set_match(flags | REJ(q), r)
            h.set_transport(0)
            c0 = h.launch_count()
            on = h.recognise(pcm, 2400)
            n_launch = h.launch_count() - c0
            assert [t for t, _ in h.timing_collect()] == tags_off, q
            n_rej[q] = _same_but_status(on, off, q, "host plain")
            h.set_transport(1)
            _same_but_status(h.recognise(pcm, 2400), off, q, "host packed")
            h.timing_collect()
            _same_but_status(recognise_dev_np(h, pcm, 2400, T), dev_off, q, "device")
            h.use_own_stream()
            h.set_match(flags, r)
            h.set_transport(0)
            c0 = h.launch_count()
            h.recognise(pcm, 2400)
            assert h.launch_count() - c0 == n_launch, q
            h.timing_collect()
        assert 0 < n_rej[1] <= n_rej[100] <= n_rej[1000] <= n_rej[65535] and n_rej[100] < good.sum(), n_rej
    finally:
        h.close()


@pytest.mark.gpu
def test_rule_boundary_and_runner_up_are_exact(case):
    """q chosen so that 1000 (d2 - d1) == q d1 exactly for some utterance: that decision stands (strict '<'); and every
    decision whose winner's own command holds the next slot is judged by the next command, not the next slot"""
    pcm, bank, T = case["pcm"], case["bank"], case["T"]
    h = handle(bank, T, 0, 0)
    try:
        off = h.recognise(pcm, 2400)
        good = off["status"] == OK
        s = off["score"][good].astype(np.int64)
        i1, d1, _, _ = decide(off["score"][good], 1, 1)
        d1 = d1.astype(np.int64)
        masked = np.where((np.arange(T)[None, :] // 4) == (i1 // 4)[:, None], DIS_ERR, s)
        d2 = masked.min(axis=1)
        own = np.where(np.arange(T)[None, :] == i1[:, None], DIS_ERR, s).min(axis=1)
        assert (own < d2).sum() > len(d2) // 2                     # the bank's same-command slots sit closest
        qs = sorted({int(1000 * (a - b) // b) for a, b in zip(d2, d1) if b and 1000 * (a - b) % b == 0 and
                     0 < 1000 * (a - b) // b <= 65535})
        assert qs, "no exact boundary in this batch"
        for q in qs[:6]:
            h.set_match(REJ(q), 0)
            on = h.recognise(pcm, 2400)
            _same_but_status(on, off, q, "boundary")
            exact = np.flatnonzero(good)[(1000 * (d2 - d1) == q * d1) & (d1 > 0)]
            assert (on["status"][exact] == OK).all(), q
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", (1, 2, 5, 80, 1024))
def test_bank_widths_and_batch_edges(T):
    """banks of 1, 2, 5, 80 and 1024 slots (one thread per utterance up to 32 commands, a warp beyond), batches just
    below, at and above multiples of the scan's rows (132 and 2112 utterances), under the greedy walk and each band
    kernel: the rule-on device call equals the rule-off one except where the rule says"""
    bank = _bank_of(T, 0x7E3B0000 + T)
    h = handle(bank, T, 0, 0)
    try:
        for B in ((131, 132, 133) if T != 1024 else (131, 2113)):
            pcm = sr_b200.synth_pcm_host(B, U, 0x7E360000 + B, 2)
            for flags, r in ((0, 0), (BAND, 5), (BAND, 10), (BAND, 16), (SYM, 10)):
                h.set_match(flags, r)
                off = recognise_dev_np(h, pcm, 2400, T)
                h.use_own_stream()
                for q in (100, 65535):
                    h.set_match(flags | REJ(q), r)
                    n = _same_but_status(recognise_dev_np(h, pcm, 2400, T), off, q, (T, B, flags, r))
                    h.use_own_stream()
                    if T <= 4:
                        assert n == 0                                # one command: nothing to compare with
    finally:
        h.close()


# ---- long recordings and streams ------------------------------------------------------------------------------------------
def _cmp_long_rule(on, off, want, what):
    """on's records are want's, and want's are the rule-off records off except status (the rule's decision is the
    nearest slot's); the number of rejections"""
    assert np.array_equal(on["n_segs"], off["n_segs"]), what
    kept = want["segs"].copy()
    kept["status"] = off["segs"]["status"]
    assert kept.tobytes() == off["segs"].tobytes(), what
    for b in range(len(off["n_segs"])):
        m = min(int(off["n_segs"][b]), off["segs"].shape[1])
        assert np.array_equal(on["segs"][b, :m]["status"], want["segs"][b, :m]["status"]), (what, b)
        assert on["segs"][b, :m].tobytes() == want["segs"][b, :m].tobytes(), (what, b)
    return int((want["segs"]["status"] == REJECT).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", ((0, 0), (BAND, 10), (RATE, 118), (SYM, 10)), ids=lambda m: "%d_r%d" % m)
def test_long_batch_and_dev_under_the_rule(matcher):
    """sr_recognise_long_batch and its _dev form: the rule-on records equal the rule-off ones except status, which is
    SR_ST_REJECT exactly where the rule on the oracle's scores says; same launches and tags"""
    flags, r = matcher
    lens = np.array([70001, 161, 123457, 99999, 200000], np.uint32)
    pcm = synth_long_poisoned(lens, 200000, 0x7E40)
    bank, T = _bank_of(40, 0x7E3C0000), 40
    h = handle(bank, T, flags, r)
    try:
        h.timing_enable(64)
        off = h.recognise_long_batch(pcm, 64, 2400, lens)
        tags = [t for t, _ in h.timing_collect()]
        total = 0
        for q in (100, 1000):
            h.set_match(flags | REJ(q), r)
            want = ox.long_under_rule(off, pcm, 2400, lens, bank, T, matcher, 1, q)
            on = h.recognise_long_batch(pcm, 64, 2400, lens)
            assert [t for t, _ in h.timing_collect()] == tags
            total += _cmp_long_rule(on, off, want, "host")
            got = recognise_long_dev_np(h, pcm, lens, 64)
            h.timing_collect()
            _cmp_long_rule(got, off, want, "dev")
        assert total > 0
    finally:
        h.close()


@pytest.mark.gpu
def test_k4_streams_under_the_rule():
    """fixed-capture pools, ragged pushes, the rule switched between pushes (off, q = 100, q = 1000): every event equals
    the rule-off pool's event except status, which is SR_ST_REJECT exactly where the rule on the oracle's scores says"""
    S, L = 24, 40000
    bank, T = _bank_of(40, 0x7E3D0000), 40
    pcm = sr_b200.synth_pcm_host(S, L, 0x7E370000, 3)
    pcm[3] = 2048
    runs = {}
    for label, qs in (("off", None), ("on", (0, 100, 1000))):
        h = handle(bank, T, BAND, 10)
        try:
            pool = sr_b200.StreamPool(h, S, L, 2400)

            def on_push(p, qs=qs, h=h):
                if qs is None:
                    return 0
                q = qs[p % 3]
                h.set_match(BAND | REJ(q), 10)
                return q
            runs[label] = k4_events(pool, pcm, "ragged", np.random.default_rng(0x7E4), on_push)
            seg, atap = pool.segments()
            pool.close()
        finally:
            h.close()
    off = {event_key(e): e for e, _ in runs["off"]}
    assert sorted(off) == sorted(event_key(e) for e, _ in runs["on"])
    ora, n_rej = ob.best_oracle(), 0
    for e, q in runs["on"]:
        o = off[event_key(e)]
        for k in ("start", "end", "frm_num", "best_idx", "best_dis", "cmd"):
            assert e[k] == o[k], (k, e, o)
        want = o["status"]
        if want == OK and q:
            s, k = event_key(e)
            f = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
            sc = ox.match_scores(f, bank, T, BAND, 10)
            idx, d1, _, rej = decide(sc, 1, q)
            assert (idx[0], d1[0]) == (o["best_idx"], o["best_dis"])
            want = REJECT if rej[0] else OK
        assert e["status"] == want, (e, o, q)
        n_rej += want == REJECT
    assert n_rej > 0


@pytest.mark.gpu
def test_k14_rule_switched_between_pushes():
    """a live long-stream pool with the rule switched between pushes (q = 0, 100, 65535): every event equals the same
    pool's event without the rule except status, which is the rule's on the oracle's scores"""
    xs = list(ox.synth_long(4, 160000, 0x7E50))
    bank, T = _bank_of(40, 0x7E3E0000), 40
    runs = {}
    for label, qs in (("off", None), ("on", (0, 100, 65535))):
        h = handle(bank, T, 0, 0)
        try:
            pool = sr_b200.LongStreamPool(h, len(xs), 3000, 2400)

            def on_push(p, qs=qs, h=h):
                if qs is None:
                    return 0
                q = qs[p % 3]
                h.set_match(REJ(q), 0)
                return q
            runs[label] = k14_events(pool, xs, 3000, on_push)
            pool.close()
        finally:
            h.close()
    off = {event_key(e): e for e, _ in runs["off"]}
    assert sorted(off) == sorted(event_key(e) for e, _ in runs["on"])
    Ul = max(len(x) for x in xs)
    pcm = np.zeros((len(xs), Ul), np.uint16)
    lens = np.array([len(x) for x in xs], np.uint32)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    w = ox.recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, 0, 4096, 256, lens)
    n_rej, seen_q = 0, set()
    for e, q in runs["on"]:
        o = off[event_key(e)]
        for k in ("start", "end", "frm_num", "best_idx", "best_dis", "cmd"):
            assert e[k] == o[k], (k, e, o)
        want = o["status"]
        if want == OK and q:
            s = int(e["stream"])
            f = ox.ftr_of_segments(ob.port(), pcm, w["atap"], [(s, int(e["start"]), int(e["end"]))])
            sc = ox.match_scores(f, bank, T, 0, 0)
            want = REJECT if decide(sc, 1, q)[3][0] else OK
        assert e["status"] == want, (e, o, q)
        n_rej += want == REJECT
        seen_q.add(q)
    assert n_rej > 0 and seen_q == {0, 100, 65535}


# ---- unequal rules, threads -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_multi_and_groups_refuse_unequal_rules(case):
    """the rule is part of the matcher: sr_recognise_batch_multi and a stream group refuse handles whose rules differ
    (the greedy walk included, whose radius is otherwise ignored), with no launch; equal rules run"""
    import torch
    bank, T, pcm = case["bank"], case["T"], case["pcm"][:64]
    two = torch.cuda.device_count() > 1
    a = handle(bank, T, REJ(100), 0)
    b = sr_b200.Handle(1 if two else 0)
    b.set_bank(bank, T, 4096)
    try:
        for other in (0, REJ(101), BAND | REJ(100)):
            b.set_match(other, 0)
            ca, cb = a.launch_count(), b.launch_count()
            with pytest.raises(sr_b200.SrError):
                sr_b200.recognise_multi([a, b], pcm, 2400)
            assert (a.launch_count(), b.launch_count()) == (ca, cb)
        b.set_match(REJ(100), 5)                                       # the greedy walk ignores the radius
        out = sr_b200.recognise_multi([a, b], pcm, 2400)
        ref = a.recognise(pcm, 2400)
        assert np.array_equal(out["status"], ref["status"]) and np.array_equal(out["score"], ref["score"])
        if two:
            b.set_match(REJ(7), 0)
            pool = sr_b200.StreamPool([a, b], 4, 20000, 2400)
            with pytest.raises(sr_b200.SrError):
                pool.push(np.full((4, 800), 2048, np.uint16))
            pool.close()
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_two_threads_with_different_rules(case):
    """two handles on one GPU, q = 100 and q = 65535, recognising concurrently from two threads: each result equals its
    handle's result alone"""
    bank, T, pcm = case["bank"], case["T"], case["pcm"][:300]
    hs = [handle(bank, T, BAND | REJ(q), 10) for q in (100, 65535)]
    try:
        alone = [h.recognise(pcm, 2400) for h in hs]
        assert not np.array_equal(alone[0]["status"], alone[1]["status"])
        got = [[None] * 4 for _ in hs]
        errs = []

        def run(i):
            try:
                for k in range(4):
                    got[i][k] = hs[i].recognise(pcm, 2400)
            except Exception as e:                                       # reported below
                errs.append(e)
        th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        for i in range(2):
            for g in got[i]:
                for k in ("score", "best_idx", "best_dis", "cmd", "status"):
                    assert np.array_equal(g[k], alone[i][k]), (i, k)
    finally:
        for h in hs:
            h.close()
