"""The K-nearest-neighbour decision rule SR_DTW_KNN(k) (an extension: the reference decides by the one nearest slot) on
every recognition call that reads the handle's matcher.

CPU: the header and the binding define the rule; a vectorised numpy reference of the rule and of the margin rule on top
of it equals a brute force over random score rows, and KNN(1) equals the nearest-slot decision; a planted bank on which
the nearest slot names the wrong command and KNN(3) the right one, and on which the margin rule's verdict turns with the
rule, from the composed oracle's scores. GPU: the setter's flag rules; sr_dtw_batch* ignore bits 8-10; every recognition
path (host plain and packed, _dev, _multi, the long-form host and _dev calls, fixed-capture pools and live long streams)
under each matcher, k = 1 .. 4, with and without the margin rule, on banks with erased slots, a width that is not a
multiple of 4, planted ties, rows without a score and more than 32 commands, equals the numpy rule applied to the
oracle-checked scores; KNN(1) equals no rule bit for bit; bytes written; unequal rules refused by _multi.
sr_recognise_batch_dev_allgather is run on a one-rank communicator by test_decision_paths.py; stream groups over two
devices are not run here: they need two GPUs."""
import os

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import synth_long_poisoned, word_bank
from drive import cmp_long, event_key, handle, k4_events, k14_events, recognise_dev_np, recognise_long_dev_np, same
from refs import decide

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIS_ERR = 0xFFFFFFFF
BAND, SIGN, SYM, ANY = sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN, sr_b200.DTW_SYM_P1, sr_b200.DTW_ANY_RATE
RATE = BAND | ANY
KNN, REJ = sr_b200.dtw_knn, sr_b200.dtw_reject
OK, REJECT = sr_b200.ST_OK, sr_b200.ST_REJECT
# (flags, r): the greedy walk, the three band kernels (r = 5, 10, 16), any-rate at the full matrix, the symmetric DP
MATCHERS = ((0, 0), (BAND, 5), (BAND, 10), (BAND, 16), (RATE, 118), (SYM, 10))
# (k, q) of the rules tried on every path: k = 1 is the identity, q = 0 no margin rule
RULES = tuple((k, q) for k in (1, 2, 3, 4) for q in (0, 100))
U = 16000


# ---- the rule in Python --------------------------------------------------------------------------------------------------
def knn_brute(row, k, q):
    """the rule on one score row with Python integers"""
    T = len(row)
    e = []
    for c in range((T + 3) // 4):
        v = sorted(int(x) for x in row[4 * c:4 * c + 4] if x != DIS_ERR)
        m = min(k, len(v))
        e.append(sum(v[:m]) // m if m else DIS_ERR)
    c1 = min(range(len(e)), key=lambda c: (e[c], c))
    if e[c1] == DIS_ERR:
        return 0, DIS_ERR, 0, False
    own = [(int(row[t]), t) for t in range(4 * c1, min(4 * c1 + 4, T))]
    idx = min(own)[1]
    d2 = min([e[c] for c in range(len(e)) if c != c1], default=DIS_ERR)
    rej = q > 0 and d2 != DIS_ERR and 1000 * (d2 - e[c1]) < q * e[c1]
    return idx, e[c1], c1, rej


# ---- banks -----------------------------------------------------------------------------------------------------------------
# signed: every slot signed; erased: n_c < k and n_c = 0, 78 slots, ties inside a command (16 = 17) and between commands
# (command 6 = command 5); short: templates of 13 .. 20 frames, so that the longer inputs score SR_DIS_ERR against every
# slot under the 2:1 guard; wide: 38 commands (the warp-per-utterance finishers), 150 slots
BANKS = {
    "signed": lambda: (word_bank(80, 0x7E700000), 80),
    "erased": lambda: (word_bank(78, 0x7E710000, erase=(5, 6, 7, 8, 9, 10, 11, 13, 30, 31, 77),
                                  dup=((16, 17), (20, 24), (21, 25), (22, 26), (23, 27))), 78),
    "short": lambda: (word_bank(40, 0x7E720000, trunc=lambda t: 13 + t % 8), 40),
    "wide": lambda: (word_bank(150, 0x7E730000, erase=(1, 2, 3, 40, 41, 42, 43, 149)), 150),
}


def _inputs(B, seed):
    """B two-second synthetic utterances, row 3 silent (SR_ST_VAD_FAIL)"""
    pcm = sr_b200.synth_pcm_host(B, U, seed, 2)
    pcm[3] = 2048
    return pcm


def _planted():
    """eight utterances and an 8-slot bank planted around utterance 1: command 0 holds its features with noise in four
    slots, command 1 its exact features in slot 4 (score 0, the nearest slot) and three other words"""
    pcm = sr_b200.synth_pcm_host(8, U, 0x7E620000, 2)
    F = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)["ftr"]
    rng = np.random.default_rng(1)
    ftr = np.zeros(8, ob.FTR_DTYPE)
    n = int(F[1]["frm_num"])
    for k in range(4):
        ftr[k] = F[1]
        noisy = F[1]["mfcc_dat"][:n * 12].astype(np.int64) + rng.normal(0, 200, n * 12).astype(np.int64)
        ftr[k]["mfcc_dat"][:n * 12] = np.clip(noisy, -32768, 32767)
    ftr[4], ftr[5], ftr[6], ftr[7] = F[1], F[2], F[3], F[4]
    return pcm, F, sr_b200.make_bank(ftr, 4096)


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_header_and_binding_define_the_rule():
    with open(os.path.join(ROOT, "include", "speech_recog.h")) as f:
        h = f.read()
    assert "#define SR_DTW_KNN(k)     ((uint32_t)(k) << 8)" in h
    assert [KNN(k) for k in range(5)] == [0, 0x100, 0x200, 0x300, 0x400]
    for bad in (-1, 5, 7):
        with pytest.raises(ValueError):
            KNN(bad)


def test_rule_reference_equals_brute_force():
    """random rows with SR_DIS_ERR, ties and widths that are not multiples of 4: refs.decide == knn_brute, and k = 0
    and k = 1 are the nearest-slot argmin"""
    rng = np.random.default_rng(0x7E7)
    for T in (1, 3, 4, 5, 8, 13, 80, 150):
        for kind in range(3):
            hi = (5, 1000, 1 << 31)[kind]
            sc = rng.integers(0, hi, (200, T)).astype(np.uint32)
            sc[rng.random((200, T)) < 0.3] = DIS_ERR
            sc[:5] = DIS_ERR
            for k in (0, 1, 2, 3, 4):
                for q in (0, 1, 100, 65535):
                    got = decide(sc, k, q)
                    for i in range(0, 200, 7):
                        want = knn_brute(sc[i], max(k, 1), q)
                        assert tuple(int(np.asarray(g)[i]) for g in got) == tuple(int(w) for w in want), (T, k, q, i)
            nn = np.argmin(sc, axis=1)
            for k in (0, 1):
                idx, dis, _, _ = decide(sc, k)
                assert np.array_equal(idx, nn) and np.array_equal(dis, sc[np.arange(200), nn])


def _planted_scores():
    pcm, F, bank = _planted()
    return pcm, bank, ox.match_scores(F[1:2], bank, 8, 0, 0)[0]


def test_planted_case_turns_the_decision():
    """on the oracle's scores: the nearest slot names command 1, KNN(3) command 0; with q just above KNN(3)'s margin the
    margin rule rejects the KNN decision, while the nearest-slot decision (score 0) always stands"""
    _, _, sc = _planted_scores()
    assert decide(sc[None], 0)[2][0] == 1 and decide(sc[None], 3)[2][0] == 0, sc.tolist()
    d1 = int(decide(sc[None], 3)[1][0])
    d2 = (int(sc[4]) + sorted(int(x) for x in sc[5:8])[0] + sorted(int(x) for x in sc[5:8])[1]) // 3
    q = 1000 * (d2 - d1) // d1 + 1
    assert 0 < q <= 65535, (d1, d2)
    assert decide(sc[None], 3, q)[3][0] and not decide(sc[None], 0, q)[3][0]
    assert not decide(sc[None], 3, q - 1)[3][0]


# ---- GPU: setter and flag rules ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_match_rules_with_knn():
    """KNN(1..4) with every matcher, with and without REJ(q), round-trips; field values 5-7, stray bits 4-7 and 11-15 and
    the values refused before are refused, and a refused call leaves the setting unchanged"""
    h = sr_b200.Handle(0)
    try:
        for flags, r in MATCHERS:
            for k in (0, 1, 2, 3, 4):
                for q in (0, 100, 65535):
                    h.set_match(flags | KNN(k) | REJ(q), r)
                    assert h.match() == (flags | KNN(k) | REJ(q), r)
        h.set_match(SYM | KNN(3) | REJ(77), 7)
        bad = [(flags | (f << 8) | extra, r) for flags, r in MATCHERS for f in (5, 6, 7) for extra in (0, REJ(5))]
        bad += [(flags | KNN(k) | (1 << b), r) for flags, r in MATCHERS[:2] for k in (0, 2) for b in (4, 5, 6, 7, 11, 12, 15)]
        bad += [(16 | REJ(5), 3), (0x8000 | REJ(5), 3), (SYM | 8, 3), (8, 3), (BAND | 4, 3), (SIGN | KNN(2), 3),
                (ANY | KNN(2), 3), (BAND | KNN(2), -1)]
        for flags, r in bad:
            with pytest.raises(sr_b200.SrError):
                h.set_match(flags, r)
            assert h.match() == (SYM | KNN(3) | REJ(77), 7), hex(flags)
    finally:
        h.close()


@pytest.mark.gpu
def test_dtw_batch_ignores_knn_bits():
    """sr_dtw_batch and sr_dtw_batch_dev with bits 8-10 set return exactly what they return without them"""
    import torch
    bank, T = BANKS["erased"]()
    h = handle(bank, T)
    try:
        pcm = _inputs(40, 0x7E740000)
        front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
        fin = front["ftr"][front["status"] == OK]
        B = len(fin)
        dev = torch.device("cuda:0")
        d_in = torch.from_numpy(fin.view(np.uint8).copy()).to(dev)

        def dev_call(flags, r):
            out = [torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device=dev) for n in (B * T, B, B)]
            h.dtw_dev(d_in.data_ptr(), B, flags, r, *[t.data_ptr() for t in out])
            h.sync()
            return [t.cpu().numpy() for t in out]
        for flags, r in MATCHERS:
            for sign in (0, SIGN):
                base = h.dtw(fin, flags | sign, r)
                base_dev = dev_call(flags | sign, r)
                for bits in (KNN(1), KNN(3), KNN(4), 5 << 8, 7 << 8):
                    got = h.dtw(fin, flags | sign | bits, r)
                    assert all(np.array_equal(a, b) for a, b in zip(got, base)), (flags, sign, bits)
                    got = dev_call(flags | sign | bits, r)
                    assert all(np.array_equal(a, b) for a, b in zip(got, base_dev)), (flags, sign, bits)
    finally:
        h.close()


# ---- GPU: recognition under the rule ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def batch():
    pcm = _inputs(300, 0x7E750000)
    return pcm, ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)


@pytest.mark.gpu
@pytest.mark.parametrize("bank_kind", sorted(BANKS))
@pytest.mark.parametrize("matcher", MATCHERS, ids=lambda m: "%d_r%d" % m)
def test_recognise_paths_under_knn(batch, bank_kind, matcher):
    """the no-rule host call equals the oracle's scores; then for every (k, q): the host call on the plain and packed
    transport and sr_recognise_batch_dev equal the numpy rule on those scores, KNN(1) equals the call without KNN bit for
    bit, and launches and timing tags are the no-rule call's"""
    flags, r = matcher
    pcm, front = batch
    bank, T = BANKS[bank_kind]()
    good = front["status"] == OK
    sc = ox.match_scores(front["ftr"][good], bank, T, flags, r)
    if bank_kind == "short" and flags != RATE:
        assert (sc == DIS_ERR).all(axis=1).any() and not (sc == DIS_ERR).all(), "rows without a score and rows with one"
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
        plain = {}
        for k, q in RULES:
            h.set_match(flags | KNN(k) | REJ(q), r)
            want = ox.under_rule(off, k, q)
            h.set_transport(0)
            on = h.recognise(pcm, 2400)
            assert [t for t, _ in h.timing_collect()] == tags_off, (k, q)
            same(on, want, ("host plain", k, q))
            h.set_transport(1)
            same(h.recognise(pcm, 2400), want, ("host packed", k, q))
            h.timing_collect()
            same(recognise_dev_np(h, pcm, 2400, T), ox.under_rule(dev_off, k, q), ("device", k, q))
            h.use_own_stream()
            h.timing_collect()
            plain[k, q] = on
        for q in (0, 100):                                   # KNN(1) is the call without KNN, bit for bit
            h.set_match(flags | REJ(q), r)
            h.set_transport(0)
            ref = h.recognise(pcm, 2400)
            for key in ref:
                assert np.asarray(ref[key]).tobytes() == np.asarray(plain[1, q][key]).tobytes(), (q, key)
    finally:
        h.close()


@pytest.mark.gpu
def test_planted_case_on_the_gpu():
    """the planted bank: the nearest slot names command 1, KNN(3) command 0; the margin rule at the q of
    test_planted_case_turns_the_decision rejects under KNN(3) only"""
    pcm, bank, sc = _planted_scores()
    d1 = int(decide(sc[None], 3)[1][0])
    d2 = (int(sc[4]) + sum(sorted(int(x) for x in sc[5:8])[:2])) // 3
    q = 1000 * (d2 - d1) // d1 + 1
    h = handle(bank, 8)
    try:
        nn = h.recognise(pcm, 2400)
        assert nn["cmd"][1] == 1 and nn["best_idx"][1] == 4 and nn["best_dis"][1] == 0
        for k, qq, cmd, st in ((3, 0, 0, OK), (3, q, 0, REJECT), (0, q, 1, OK)):
            h.set_match(KNN(k) | REJ(qq), 0)
            out = h.recognise(pcm, 2400)
            same(out, ox.under_rule(nn, k, qq), (k, qq))
            assert (out["cmd"][1], out["status"][1]) == (cmd, st), (k, qq)
    finally:
        h.close()


@pytest.mark.gpu
def test_bytes_written_under_knn(batch):
    """sr_recognise_batch_dev outputs prefilled with 0x5A and with 0xA5: under KNN(3) | REJ(100) the decision fields come
    back equal from both fills (every byte written), and the fields the rule leaves alone are, byte for byte, what the
    no-rule call leaves in the same fill (ftr keeps the fill past its rows and in save_sign, with or without the rule)"""
    import torch
    pcm, _ = batch
    pcm = pcm[:140]
    bank, T = BANKS["wide"]()
    h = handle(bank, T, BAND, 10)
    dev = torch.device("cuda:0")
    B = pcm.shape[0]

    def run(fill):
        pcm_d = torch.from_numpy(pcm.view(np.int16)).to(dev)
        sizes = {"atap": B * 12, "seg_off": B * 24, "ftr": B * sr_b200.FTR_BYTES, "score": B * T * 4, "status": B,
                 "best_idx": B * 4, "best_dis": B * 4, "cmd": B * 4}
        out = {key: torch.full((n,), fill, dtype=torch.uint8, device=dev) for key, n in sizes.items()}
        h.recognise_dev(pcm_d.data_ptr(), pcm.shape[1], B, 2400, **{key: v.data_ptr() for key, v in out.items()})
        h.sync()
        return {key: v.cpu().numpy().tobytes() for key, v in out.items()}
    try:
        off = {fill: run(fill) for fill in (0x5A, 0xA5)}
        h.set_match(BAND | KNN(3) | REJ(100), 10)
        on = {fill: run(fill) for fill in (0x5A, 0xA5)}
        for key in ("best_idx", "best_dis", "cmd", "status"):
            assert on[0x5A][key] == on[0xA5][key], key
        for fill in (0x5A, 0xA5):
            for key in ("atap", "seg_off", "ftr", "score"):
                assert on[fill][key] == off[fill][key], (fill, key)
        assert on[0x5A]["best_dis"] != off[0x5A]["best_dis"]   # the rule's best_dis is a mean of k scores
    finally:
        h.close()


@pytest.mark.gpu
def test_multi_under_knn_and_refusal_of_unequal_rules(batch):
    """sr_recognise_batch_multi over two handles with KNN(3) | REJ(100) equals the numpy rule; handles whose KNN values
    differ are refused with no launch"""
    pcm, _ = batch
    pcm = pcm[:128]
    bank, T = BANKS["erased"]()
    a = handle(bank, T, KNN(3) | REJ(100), 0)
    b = handle(bank, T, KNN(3) | REJ(100), 5)                # the greedy walk ignores the radius
    try:
        off = handle(bank, T)
        ref = off.recognise(pcm, 2400)
        off.close()
        out = sr_b200.recognise_multi([a, b], pcm, 2400)
        want = ox.under_rule(ref, 3, 100)
        for key in out:
            assert np.array_equal(np.asarray(out[key]), np.asarray(want[key])), key
        for other in (0, KNN(2) | REJ(100), KNN(3), KNN(1) | REJ(100), BAND | KNN(3) | REJ(100)):
            b.set_match(other, 0)
            ca, cb = a.launch_count(), b.launch_count()
            with pytest.raises(sr_b200.SrError):
                sr_b200.recognise_multi([a, b], pcm, 2400)
            assert (a.launch_count(), b.launch_count()) == (ca, cb)
    finally:
        a.close()
        b.close()


# ---- long recordings and streams ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("matcher", ((0, 0), (BAND, 10), (SYM, 10)), ids=lambda m: "%d_r%d" % m)
def test_long_batch_and_dev_under_knn(matcher):
    """sr_recognise_long_batch and its _dev form under KNN(k) | REJ(q) equal the no-rule records with the rule applied to
    the oracle's scores of each OK segment; KNN(1) equals no rule"""
    flags, r = matcher
    lens = np.array([70001, 161, 123457, 99999, 200000], np.uint32)
    pcm = synth_long_poisoned(lens, 200000, 0x7E40)
    bank, T = BANKS["erased"]()
    h = handle(bank, T, flags, r)
    try:
        off = h.recognise_long_batch(pcm, 64, 2400, lens)
        changed = 0
        for k, q in ((1, 0), (2, 0), (3, 100), (4, 0), (4, 1000)):
            h.set_match(flags | KNN(k) | REJ(q), r)
            want = ox.long_under_rule(off, pcm, 2400, lens, bank, T, matcher, k, q)
            cmp_long(h.recognise_long_batch(pcm, 64, 2400, lens), want)
            cmp_long(recognise_long_dev_np(h, pcm, lens, 64), want)
            if k == 1 and q == 0:
                cmp_long(off, want)
            changed += int((want["segs"]["best_dis"] != off["segs"]["best_dis"]).sum())
        assert changed > 0
    finally:
        h.close()


# the settings a stream's pushes cycle through
STREAM_RULES = ((0, 0), (2, 0), (3, 100), (4, 0), (1, 0), (3, 0))


@pytest.mark.gpu
def test_k4_streams_under_knn_switched_between_pushes():
    """a fixed-capture pool whose KNN setting changes at every push: each event equals the rule of its push applied to
    the oracle's scores of its segment, on the same event the no-rule pool gives otherwise"""
    S, L = 24, 40000
    bank, T = BANKS["erased"]()
    pcm = sr_b200.synth_pcm_host(S, L, 0x7E370000, 3)
    pcm[3] = 2048
    h = handle(bank, T, BAND, 10)
    try:
        pool = sr_b200.StreamPool(h, S, L, 2400)

        def on_push(p):
            k, q = STREAM_RULES[p % len(STREAM_RULES)]
            h.set_match(BAND | KNN(k) | REJ(q), 10)
            return k, q
        events = k4_events(pool, pcm, "ragged", np.random.default_rng(0x7E4), on_push)
        seg, atap = pool.segments()
        pool.close()
    finally:
        h.close()
    ora, seen = ob.best_oracle(), set()
    assert len(events) >= 2 * S
    for e, (k, q) in events:
        s, j = event_key(e)
        f = ora.mfcc_batch(pcm[s:s + 1], seg[s, j].reshape(1, 2), atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]), e
        if e["frm_num"] == 0:
            assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (2, 0, DIS_ERR, 0), e
            continue
        idx, dis, cmd, rej = decide(ox.match_scores(f, bank, T, BAND, 10), k, q)
        assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (REJECT if rej[0] else OK, idx[0], dis[0], cmd[0]), \
            (k, q, e)
        seen.add((k, q))
    assert len(seen) >= 4, seen


@pytest.mark.gpu
def test_k14_streams_under_knn_switched_between_pushes():
    """a live long-stream pool whose KNN setting changes at every push: each event equals the rule of its push applied to
    the oracle's scores of its segment"""
    xs = list(ox.synth_long(4, 160000, 0x7E50))
    bank, T = BANKS["wide"]()
    h = handle(bank, T, 0, 0)
    try:
        pool = sr_b200.LongStreamPool(h, len(xs), 3000, 2400)

        def on_push(p):
            k, q = STREAM_RULES[p % len(STREAM_RULES)]
            h.set_match(KNN(k) | REJ(q), 0)
            return k, q
        events = k14_events(pool, xs, 3000, on_push)
        pool.close()
    finally:
        h.close()
    Ul = max(len(x) for x in xs)
    pcm = np.zeros((len(xs), Ul), np.uint16)
    lens = np.array([len(x) for x in xs], np.uint32)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    w = ox.recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, T, 4096, 256, lens)
    seen = set()
    for e, (k, q) in events:
        s, j = event_key(e)
        rec = w["segs"][s, j]
        assert (int(e["start"]), int(e["end"]), int(e["frm_num"])) == (int(rec["start"]), int(rec["end"]), int(rec["frm_num"]))
        if rec["status"] != OK:
            assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (rec["status"], 0, DIS_ERR, 0), e
            continue
        f = ox.ftr_of_segments(ob.port(), pcm, w["atap"], [(s, int(e["start"]), int(e["end"]))])
        idx, dis, cmd, rej = decide(ox.match_scores(f, bank, T, 0, 0), k, q)
        assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (REJECT if rej[0] else OK, idx[0], dis[0], cmd[0]), \
            (k, q, e)
        seen.add((k, q))
    assert len(seen) >= 4 and len(events) > 3 * len(xs), (seen, len(events))
