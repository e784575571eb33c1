"""The recognition decision on the paths the rule, KNN and lifter tests do not reach: the all-gather on a one-rank
communicator, the finishers' one-thread and warp forms on either side of 32 commands, the dynamic greedy scan under the
rules, the margin rule past 2^31, and the matcher flags' decode over every value of bits 0-15.

CPU: the flag model reads its constants from the header and refuses what the header says fails; the finisher banks hold
32 or 33 commands with empty commands and ties; the headroom bank's scores are all above 32 768, so q d1 passes 2^31 at
q = 65 535, and its batch holds an exact margin boundary 1000 (d2 - d1) = q d1.
GPU: sr_recognise_batch_dev_allgather on a world of one rank under each matcher (greedy static and dynamic, band r = 5,
10, 16, any-rate r = 118, symmetric r = 10), with no rule, REJECT, KNN and both, each with and without the lifter:
gathered scores are the call's scores and gathered keys best_dis << 32 | best_idx of the oracle's decision on every row;
back-to-back calls that grow the key buffer, a gather of the keys alone and a plain sr_recognise_batch_dev between two
gathers keep their results apart; sr_allgather_dev copies a buffer. Banks of 125, 128, 129 and 132 slots under four rules
through recognise (host plain and packed, _dev), the long-form calls (host, _dev), a lock-step fixed-capture pool and a
live long-stream pool. The dynamic greedy scan under KNN | REJECT, with and without the lifter, equals the static one
bit for bit and the oracle on recognise, _dev, the long-form calls and a fixed-capture pool. The margin rule at q =
65 535 and at the exact boundary on the headroom bank. sr_set_match, sr_get_match and sr_dtw_batch_dev over every value
of bits 0-15 against the model. Every expected record comes from the oracle compositions (oracle_ext, lifter_ref) and
refs.decide."""
import os
import re

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import bank_planted, headroom_bank, inputs, synth_long_poisoned, word_bank
from drive import (check_k4, check_k14, cmp_long, handle, k4_events, k14_events, long_records, recognise_dev_launch,
                   recognise_dev_np, recognise_dev_read, recognise_long_dev_np, same)
from lifter_ref import compose_recognise
from refs import decide

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIS_ERR = 0xFFFFFFFF
BAND, SIGN, SYM, ANY, LIFT = sr_b200.DTW_BAND, sr_b200.DTW_CHECK_SIGN, sr_b200.DTW_SYM_P1, sr_b200.DTW_ANY_RATE, sr_b200.DTW_LIFTER
RATE = BAND | ANY
KNN, REJ = sr_b200.dtw_knn, sr_b200.dtw_reject
OK, VAD_FAIL, MFCC_FAIL, REJECT = sr_b200.ST_OK, sr_b200.ST_VAD_FAIL, sr_b200.ST_MFCC_FAIL, sr_b200.ST_REJECT
U = 16000
# (flags, r, dtw variant) of the all-gather: the greedy walk on the static and the dynamic scan, the three band kernels,
# any-rate at the full matrix, the symmetric DP
GATHER_MATCHERS = ((0, 0, 0), (0, 0, 1), (BAND, 5, 0), (BAND, 10, 0), (BAND, 16, 0), (RATE, 118, 0), (SYM, 10, 0))
# (k, q) of the all-gather: no rule, the margin rule, KNN, both; each with and without the lifter
GATHER_RULES = ((0, 0), (0, 100), (3, 0), (2, 100))
# (k, q, lifter) of the finisher widths
WIDTH_RULES = ((0, 100, 0), (2, 0, 0), (3, 100, 0), (4, 0, LIFT))


def _ids(m):
    return "_".join(str(x) for x in m)


def _key(rec):
    """best_dis << 32 | best_idx of a recognition record"""
    return (np.asarray(rec["best_dis"]).astype(np.uint64) << np.uint64(32)) | np.asarray(rec["best_idx"]).astype(np.uint64)


# ---- the flag decode, modelled from the header's text -------------------------------------------------------------------
def _header_defines():
    with open(os.path.join(ROOT, "include", "speech_recog.h")) as f:
        h = f.read()
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (SR_DTW_\w+)\s+(\d+)u\b", h)}
    d["SR_DTW_LIFTER"] = 1 << int(re.search(r"#define SR_DTW_LIFTER\s+\(1u << (\d+)\)", h).group(1))
    d["KNN_SHIFT"] = int(re.search(r"#define SR_DTW_KNN\(k\)\s+\(\(uint32_t\)\(k\) << (\d+)\)", h).group(1))
    d["REJECT_SHIFT"] = int(re.search(r"#define SR_DTW_REJECT\(q\)\s+\(\(uint32_t\)\(q\) << (\d+)\)", h).group(1))
    d["FTR_PER_COMM"] = int(re.search(r"#define SR_FTR_PER_COMM\s+(\d+)u", h).group(1))
    return d


HDR = _header_defines()
# the four matchers of sr_set_match: the greedy walk, SR_DTW_BAND, SR_DTW_BAND | SR_DTW_ANY_RATE, SR_DTW_SYM_P1
MATCHER_WORDS = {0, HDR["SR_DTW_BAND"], HDR["SR_DTW_BAND"] | HDR["SR_DTW_ANY_RATE"], HDR["SR_DTW_SYM_P1"]}
MATCHER_BITS = HDR["SR_DTW_BAND"] | HDR["SR_DTW_SYM_P1"] | HDR["SR_DTW_ANY_RATE"]
KNN_FIELD = 7 << HDR["KNN_SHIFT"]


def set_match_accepts(w, r):
    """sr_set_match(w, r) per the header: one of the four matchers (SR_DTW_CHECK_SIGN is the recognition calls' own),
    a KNN field of 0..SR_FTR_PER_COMM, SR_DTW_LIFTER, any q in bits 16-31, no other bit in 4-15, and band_r >= 0"""
    knn = (w & KNN_FIELD) >> HDR["KNN_SHIFT"]
    stray = w & 0xFFF0 & ~KNN_FIELD & ~HDR["SR_DTW_LIFTER"]
    return (w & 0xF) in MATCHER_WORDS and knn <= HDR["FTR_PER_COMM"] and not stray and r >= 0


def dtw_batch_accepts(w, r):
    """sr_dtw_batch_dev(w, r) per the header: one of the four matchers, SR_DTW_CHECK_SIGN allowed; no bit >= 16; bits
    4-15 other than SR_DTW_LIFTER accepted and ignored; a DP's band_r >= 0 (the greedy walk has none)"""
    m = w & MATCHER_BITS
    return m in MATCHER_WORDS and w >> 16 == 0 and (m == 0 or r >= 0)


def dtw_batch_effective(w):
    """the flags sr_dtw_batch_dev acts on: the matcher, SR_DTW_CHECK_SIGN and SR_DTW_LIFTER"""
    return w & (0xF | HDR["SR_DTW_LIFTER"])


def test_flag_model_reads_the_header():
    """the model's constants are the header's and the binding's, and it refuses what the header says fails"""
    assert (HDR["SR_DTW_CHECK_SIGN"], HDR["SR_DTW_BAND"], HDR["SR_DTW_SYM_P1"], HDR["SR_DTW_ANY_RATE"],
            HDR["SR_DTW_LIFTER"]) == (SIGN, BAND, SYM, ANY, LIFT)
    assert (1 << HDR["KNN_SHIFT"], 1 << HDR["REJECT_SHIFT"]) == (KNN(1), REJ(1)) and HDR["FTR_PER_COMM"] == 4
    for w in (SYM | BAND, ANY, SYM | ANY, SIGN, KNN(4) + (1 << 8), 7 << 8, 1 << 4, 1 << 15, 1 << 11, 1 << 12):
        assert not set_match_accepts(w, 0), hex(w)
    for w in (0, BAND, RATE, SYM, SYM | KNN(4) | LIFT | REJ(65535), BAND | KNN(1) | REJ(1)):
        assert set_match_accepts(w, 0) and not set_match_accepts(w, -1), hex(w)
    assert dtw_batch_accepts(SIGN | BAND | (5 << 8) | (1 << 15), 0) and not dtw_batch_accepts(BAND | REJ(1), 0)
    assert dtw_batch_accepts(SIGN | (1 << 4), -1) and not dtw_batch_accepts(SYM, -1) and not dtw_batch_accepts(SYM | BAND, 3)


@pytest.mark.gpu
def test_set_match_over_every_low_word():
    """sr_set_match at every value of bits 0-15, at r = -1, 0, 10, 118, 2^31 - 1 and q = 0, 1, 65 535: accepted exactly
    where the model says; sr_get_match returns the word as set, and after a refusal the setting before it"""
    import ctypes as C
    L = sr_b200.lib()
    h = sr_b200.Handle(0)
    try:
        f, rr = C.c_uint32(0), C.c_int(0)
        cur = (0, 0)
        bad = []
        for r in (-1, 0, 10, 118, 2 ** 31 - 1):
            for q in (0, 1, 65535):
                for low in range(1 << 16):
                    w = low | q << 16
                    ok = L.sr_set_match(h._h, w, r) == 0
                    if ok:
                        cur = (w, r)
                    L.sr_get_match(h._h, C.byref(f), C.byref(rr))
                    if ok != set_match_accepts(w, r) or (f.value, rr.value) != cur:
                        bad.append((hex(w), r, ok, (f.value, rr.value), cur))
        assert not bad, (len(bad), bad[:8])
    finally:
        h.close()


@pytest.mark.gpu
def test_dtw_batch_dev_over_every_low_word():
    """sr_dtw_batch_dev at every value of bits 0-15 (r = 10 and r = -1) on a tiny batch against a bank with erased,
    unsigned and over-long slots: refused exactly where the model says, and where accepted its scores, best_idx and
    best_dis are those of the word with the ignored bits cleared"""
    import torch
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0xF1A6)
    T, B = 12, 3
    bank = bank_planted(rng, T)
    fin = inputs(rng, [9, 30, 61])
    h = handle(bank, T)
    try:
        d_in = torch.from_numpy(fin.view(np.uint8).copy()).to(dev)
        words = [(w, r) for r in (10, -1) for w in range(1 << 16)]
        per = B * T + 2 * B
        out = torch.full((len(words) * per,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        base = out.data_ptr()
        refused = set()
        for n, (w, r) in enumerate(words):
            p = base + 4 * n * per
            try:
                h.dtw_dev(d_in.data_ptr(), B, w, r, p, p + 4 * B * T, p + 4 * (B * T + B))
            except sr_b200.SrError:
                refused.add(n)
        h.sync()
        got = out.cpu().numpy().reshape(len(words), per)
        wrong = [hex(words[n][0]) for n in range(len(words)) if (n in refused) == dtw_batch_accepts(*words[n])]
        assert not wrong, (len(wrong), wrong[:8])
        untouched = np.full(per, 0x5A5A5A5A, np.int32)
        assert all(np.array_equal(got[n], untouched) for n in refused)
        index = {wr: n for n, wr in enumerate(words)}
        bad = [hex(w) for n, (w, r) in enumerate(words) if dtw_batch_accepts(w, r) and
               not np.array_equal(got[n], got[index[dtw_batch_effective(w), r]])]
        assert not bad, (len(bad), bad[:8])
        assert len({got[index[w, 10]].tobytes() for w in (0, SIGN, BAND, SYM, RATE, LIFT)}) == 6   # each bit matters
    finally:
        h.close()


# ---- the all-gather on a one-rank communicator ------------------------------------------------------------------------------
def _comm_handle(bank, T):
    """a handle with the bank and a communicator of one rank, or a skip when the library cannot load libnccl"""
    import torch  # noqa: F401  (the process's libnccl, when torch brings one)
    if sr_b200.lib().sr_comm_nccl_version() == 0:
        pytest.skip("libnccl cannot be loaded")
    h = handle(bank, T)
    try:
        h.comm_create(0, 1, sr_b200.comm_unique_id())
        assert (sr_b200.lib().sr_comm_rank(h._h), sr_b200.lib().sr_comm_world(h._h)) == (0, 1)
    except BaseException:
        h.close()
        raise
    return h


def _gather(h, pcm, T, fields=sr_b200.RECOG_FIELDS, gather=("score", "best")):
    """one sr_recognise_batch_dev_allgather on a fresh torch stream, then sr_comm_wait and a synchronise"""
    import torch
    st = torch.cuda.Stream(torch.device("cuda:0"))
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        bufs = recognise_dev_launch(h, pcm, 2400, T, fields, gather)
        h.comm_wait()
    st.synchronize()
    h.sync()
    return recognise_dev_read(bufs)


def _gathered_ok(got, want, what):
    """the call's fields equal want, its gathered scores its scores, its gathered keys want's decision keys"""
    same(got, want, what)
    assert np.array_equal(got["gathered_score"], got["score"]), what
    bad = np.flatnonzero(got["gathered_best"] != _key(want))
    assert len(bad) == 0, (what, bad[:8].tolist())


@pytest.fixture(scope="module")
def gather_case():
    """96 two-second utterances, row 3 silent (SR_ST_VAD_FAIL), row 4 a tone of more than 119 frames (SR_ST_MFCC_FAIL);
    78 slots with unsigned slots, commands with fewer than k and with no signed slot, and ties within and between commands"""
    pcm = sr_b200.synth_pcm_host(96, U, 0xA6A00000, 2)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64)
    front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
    assert front["status"][3] == VAD_FAIL and front["status"][4] == MFCC_FAIL, front["status"][:8]
    bank = word_bank(78, 0xA6A10000, erase=(5, 6, 7, 8, 9, 10, 11, 13, 30, 31, 77),
                     dup=((16, 17), (20, 24), (21, 25), (22, 26), (23, 27)))
    return pcm, front, bank, 78


@pytest.mark.gpu
@pytest.mark.parametrize("matcher", GATHER_MATCHERS, ids=_ids)
def test_allgather_one_rank_equals_the_decision(gather_case, matcher):
    """sr_recognise_batch_dev_allgather, one rank, under the matcher with each rule, with and without the lifter: every
    field equals the oracle's decision, the gathered scores the call's scores, and the gathered key of every row --
    failed and rejected ones included -- best_dis << 32 | best_idx"""
    flags, r, variant = matcher
    pcm, front, bank, T = gather_case
    h = _comm_handle(bank, T)
    try:
        h.set_dtw_variant(variant)
        seen = set()
        for lift in (0, LIFT):
            off = compose_recognise(front, bank, T, flags | lift, r)
            for k, q in GATHER_RULES:
                h.set_match(flags | lift | KNN(k) | REJ(q), r)
                want = ox.under_rule(off, k, q)
                _gathered_ok(_gather(h, pcm, T), want, (lift, k, q))
                seen |= set(want["status"].tolist())
        assert seen == {OK, VAD_FAIL, MFCC_FAIL, REJECT}, seen
    finally:
        h.close()


@pytest.mark.gpu
def test_allgather_calls_back_to_back():
    """on one torch stream with no synchronise in between: a gather with no rule, one under KNN(3) on the 150-slot bank
    (its key rows grow the key buffer), one with no rule again, then a gather of the keys alone (score and best_idx NULL),
    a plain sr_recognise_batch_dev and another gather; batches of different sizes and PCM, each with its own buffers.
    Each equals its oracle decision; then sr_allgather_dev copies a buffer of its own"""
    import torch
    bank = word_bank(150, 0xA6A20000, erase=(1, 2, 3, 40, 41, 42, 43, 149))
    T = 150
    pcms = [sr_b200.synth_pcm_host(B, U, 0xA6A30000 + B, 2) for B in (40, 71, 33, 52, 64, 45)]
    for p in pcms:
        p[1] = 2048
    fronts = [ob.recognise_pinned(ob.best_oracle(), p, 2400, None, 0, 4096) for p in pcms]
    off = [ox.compose_recognise(f, bank, T, 0, 0) for f in fronts]
    h = _comm_handle(bank, T)
    try:
        st = torch.cuda.Stream(torch.device("cuda:0"))
        h.set_stream(st.cuda_stream)
        rules = ((0, 0), (3, 0), (0, 0), (2, 100), (3, 100), (0, 100))
        keys_only = ("status", "best_dis", "cmd")
        with torch.cuda.stream(st):
            runs = []
            for n, (pcm, (k, q)) in enumerate(zip(pcms, rules)):
                h.set_match(KNN(k) | REJ(q), 0)
                if n == 3:
                    runs.append(recognise_dev_launch(h, pcm, 2400, T, keys_only, ("best",)))
                elif n == 4:
                    runs.append(recognise_dev_launch(h, pcm, 2400, T))
                else:
                    runs.append(recognise_dev_launch(h, pcm, 2400, T, gather=("score", "best")))
            h.comm_wait()
        st.synchronize()
        h.sync()
        for n, (bufs, (k, q)) in enumerate(zip(runs, rules)):
            got, want = recognise_dev_read(bufs), ox.under_rule(off[n], k, q)
            if n == 3:
                for key in keys_only:
                    assert np.array_equal(got[key], want[key]), (n, key)
                assert np.array_equal(got["gathered_best"], _key(want)), n
            elif n == 4:
                same(got, want, n)
            else:
                _gathered_ok(got, want, n)
        with torch.cuda.stream(st):
            src = torch.randint(0, 256, (1 << 20,), dtype=torch.uint8, device="cuda:0")
            dst = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda:0")
            h.allgather_dev(src.data_ptr(), dst.data_ptr(), 1 << 20)
            h.allgather_dev(None, None, 0)
            h.comm_wait()
        st.synchronize()
        assert torch.equal(src, dst)
    finally:
        h.close()


# ---- the finishers' one-thread and warp forms ---------------------------------------------------------------------------
def _width_bank(T):
    """T slots of word_bank: command 0 with one signed slot, command 10 with none, the last slot unsigned, a tie inside
    command 4 (slot 16 = slot 17) and between commands 5 and 6"""
    return word_bank(T, 0xA6B00000 + T, erase=(1, 2, 3, 40, 41, 42, 43, T - 1),
                     dup=((16, 17), (20, 24), (21, 25), (22, 26), (23, 27)))


def test_width_banks_straddle_32_commands():
    """the banks of the finisher tests hold 32, 32, 33 and 33 commands (the one-thread and the warp form), with the
    planted empty command and ties"""
    for T, n_cmd in ((125, 32), (128, 32), (129, 33), (132, 33)):
        bank = _width_bank(T)
        assert bank.shape[0] == T and (T + 3) // 4 == n_cmd
        sign = bank[:, 0].astype(int) | bank[:, 1].astype(int) << 8
        assert (sign[40:44] != sr_b200.SAVE_MASK).all() and (sign[1:4] != sr_b200.SAVE_MASK).all() and sign[0] == sr_b200.SAVE_MASK
        assert bank[16].tobytes() == bank[17].tobytes() and bank[20:24].tobytes() == bank[24:28].tobytes()


@pytest.fixture(scope="module")
def width_pcm():
    pcm = sr_b200.synth_pcm_host(140, U, 0xA6B10000, 2)
    pcm[3] = 2048
    return pcm, ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)


@pytest.mark.gpu
@pytest.mark.parametrize("T", (125, 128, 129, 132))
def test_finisher_widths_under_the_rules(width_pcm, T):
    """banks of 32 and 33 commands under REJECT(100), KNN(2), KNN(3) | REJECT(100) and KNN(4) | LIFTER: recognise on
    both transports and _dev (best_final_kernel), the long-form host and _dev calls (long_scatter_kernel, more records
    than a CTA holds in warps), a lock-step fixed-capture pool and a live long-stream pool with the rule switched at every
    push (stream_finish_kernel) equal the oracle's decisions"""
    pcm, front = width_pcm
    bank = _width_bank(T)
    lens = np.array([70001, 161, 123457, 99999], np.uint32)
    lpcm = synth_long_poisoned(lens, 123457, 0xA6B2)
    h = handle(bank, T)
    try:
        off = {lift: compose_recognise(front, bank, T, lift, 0) for lift in (0, LIFT)}
        for k, q, lift in WIDTH_RULES:
            h.set_match(lift | KNN(k) | REJ(q), 0)
            want = ox.under_rule(off[lift], k, q)
            h.set_transport(0)
            same(h.recognise(pcm, 2400), want, ("host plain", k, q, lift))
            h.set_transport(1)
            same(h.recognise(pcm, 2400), want, ("host packed", k, q, lift))
            same(recognise_dev_np(h, pcm, 2400, T), want, ("device", k, q, lift))
            h.use_own_stream()
            lw = long_records(lpcm, lens, bank, T, (lift, 0, k, q), max_segs=16)
            cmp_long(h.recognise_long_batch(lpcm, 16, 2400, lens), lw)
            cmp_long(recognise_long_dev_np(h, lpcm, lens, 16), lw)
        n_rec = int(np.minimum(lw["n_segs"], 16).sum())
        assert n_rec > 8, n_rec                     # more records than one 256-thread CTA decides at a warp per record
        rules = [(lift, 0, k, q) for k, q, lift in WIDTH_RULES]
        S, Lc = 16, 40000
        spcm = sr_b200.synth_pcm_host(S, Lc, 0xA6B30000 + T, 3)
        spcm[3] = 2048

        def on_push(p):
            m = rules[p % len(rules)]
            h.set_match(m[0] | KNN(m[2]) | REJ(m[3]), m[1])
            return m
        pool = sr_b200.StreamPool(h, S, Lc, 2400)
        events = k4_events(pool, spcm, "lockstep", None, on_push)
        check_k4(events, pool, spcm, bank, T)
        pool.close()
        xs = list(ox.synth_long(3, 120000, 0xA6B4 + T))
        lpool = sr_b200.LongStreamPool(h, len(xs), 3000, 2400)
        events = k14_events(lpool, xs, 3000, on_push)
        lpool.close()
        check_k14(events, xs, bank, T, rules)
    finally:
        h.close()


# ---- the dynamic greedy scan under the rules ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lift", (0, LIFT), ids=("plain", "lifter"))
def test_dynamic_scan_under_the_rules(gather_case, lift):
    """set_dtw_variant(1) under KNN(k) | REJECT(q): recognise (host), _dev, the long-form host and _dev calls and a
    fixed-capture pool equal the static variant (0) bit for bit, and the oracle"""
    pcm, front, bank, T = gather_case
    lens = np.array([70001, 161, 123457, 99999, 150000], np.uint32)
    lpcm = synth_long_poisoned(lens, 150000, 0xA6C0)
    S, Lc = 16, 40000
    spcm = sr_b200.synth_pcm_host(S, Lc, 0xA6C10000, 3)
    spcm[3] = 2048
    off = compose_recognise(front, bank, T, lift, 0)
    rules = ((2, 100), (3, 1000), (4, 0))
    h = handle(bank, T)
    try:
        runs = {}
        for variant in (0, 1):
            h.set_dtw_variant(variant)
            got = []
            for k, q in rules:
                h.set_match(lift | KNN(k) | REJ(q), 0)
                want = ox.under_rule(off, k, q)
                rec = h.recognise(pcm, 2400)
                same(rec, want, (variant, k, q))
                d = recognise_dev_np(h, pcm, 2400, T)
                h.use_own_stream()
                same(d, want, (variant, k, q, "device"))
                lh = h.recognise_long_batch(lpcm, 64, 2400, lens)
                ld = recognise_long_dev_np(h, lpcm, lens, 64)
                got.append((rec, d, lh, ld))

            def on_push(p):
                k, q = rules[p % len(rules)]
                h.set_match(lift | KNN(k) | REJ(q), 0)
                return (lift, 0, k, q)
            pool = sr_b200.StreamPool(h, S, Lc, 2400)
            events = k4_events(pool, spcm, "ragged", np.random.default_rng(0xA6C2), on_push)
            check_k4(events, pool, spcm, bank, T)
            pool.close()
            runs[variant] = (got, events)
        for (a, b) in zip(runs[0][0], runs[1][0]):
            for x, y in zip(a, b):
                for key in x:
                    assert np.asarray(x[key]).tobytes() == np.asarray(y[key]).tobytes(), key
        assert runs[0][1] == runs[1][1]
        for k, q in rules:
            lw = long_records(lpcm, lens, bank, T, (lift, 0, k, q), max_segs=64)
            n = rules.index((k, q))
            cmp_long(runs[1][0][n][2], lw)
            cmp_long(runs[1][0][n][3], lw)
    finally:
        h.close()


# ---- the margin rule past 2^31 ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def headroom():
    """3 000 two-second utterances against headroom_bank: for the greedy walk and the symmetric DP at r = 10, the
    oracle's scores of the OK rows and the margin boundaries (matcher, k, q, row) at which 1000 (d2 - d1) = q d1"""
    pcm = sr_b200.synth_pcm_host(3000, U, 0x7E910000, 2)
    front = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, None, 0, 4096)
    bank = headroom_bank(0x7E900000)
    T = 8
    good = front["status"] == OK
    cases = {}
    for flags, r in ((0, 0), (SYM, 10)):
        sc = ox.match_scores(front["ftr"][good], bank, T, flags, r)
        for k in (0, 2, 3, 4):
            _, d1, cmd, _ = decide(sc, k)
            runner = np.where((np.arange(T)[None, :] // 4) == cmd[:, None], DIS_ERR, sc).astype(np.uint32)
            d2 = decide(runner, k)[1].astype(np.int64)      # the other command's decision is the runner-up
            d1 = d1.astype(np.int64)
            exact = (d2 > d1) & (1000 * (d2 - d1) % d1 == 0) & (1000 * (d2 - d1) // d1 <= 65535)
            cases[flags, r, k] = dict(sc=sc, d1=d1, d2=d2, bounds=[(int(1000 * (d2[i] - d1[i]) // d1[i]), int(i))
                                                                   for i in np.flatnonzero(exact)])
    return pcm, front, bank, T, cases


def test_headroom_case_passes_2_31(headroom):
    """every score of the OK rows is above 32 768 and below SR_DIS_ERR, so 65 535 d1 > 2^31 on every decision; a
    signed 32-bit product would keep the decisions the rule rejects at q = 65 535; the batch holds an exact boundary"""
    _, _, _, _, cases = headroom
    n_bounds = 0
    for (flags, r, k), c in cases.items():
        signed = np.arange(8) != 6                                          # slot 6 is unsigned
        assert (c["sc"][:, signed] > 32768).all() and (c["sc"][:, signed] != DIS_ERR).all() and \
            (c["sc"][:, 6] == DIS_ERR).all(), (flags, k)
        assert (65535 * c["d1"] > 2 ** 31).all() and (c["d2"] != DIS_ERR).all()
        rej = decide(c["sc"], k, 65535)[3]
        wrapped = ((65535 * c["d1"] + 2 ** 31) % 2 ** 32 - 2 ** 31)         # the product in s32
        assert rej.all() and not (1000 * (c["d2"] - c["d1"]) < wrapped).any(), (flags, k)
        for q, i in c["bounds"]:
            assert 1000 * (c["d2"][i] - c["d1"][i]) == q * c["d1"][i] and not decide(c["sc"][i:i + 1], k, q)[3][0]
            assert decide(c["sc"][i:i + 1], k, q + 1)[3][0]
        n_bounds += len(c["bounds"])
    assert n_bounds > 0


@pytest.mark.gpu
def test_margin_rule_past_2_31(headroom):
    """the headroom bank under the greedy walk and the symmetric DP, k = 0, 2, 3, 4: at q = 65 535 every decision is
    rejected, and at each exact boundary q the boundary row's decision stands; every record equals the oracle's"""
    pcm, front, bank, T, cases = headroom
    h = handle(bank, T)
    try:
        for (flags, r, k), c in cases.items():
            off = ox.compose_recognise(front, bank, T, flags, r)
            ok = np.flatnonzero(front["status"] == OK)
            for q in [65535] + [q for q, _ in c["bounds"]]:
                h.set_match(flags | KNN(k) | REJ(q), r)
                got = h.recognise(pcm, 2400)
                same(got, ox.under_rule(off, k, q), (flags, k, q))
                if q == 65535:
                    assert (got["status"][ok] == REJECT).all(), (flags, k)
            for q, i in c["bounds"]:
                h.set_match(flags | KNN(k) | REJ(q), r)
                assert h.recognise(pcm[ok[i]:ok[i] + 1], 2400)["status"][0] == OK, (flags, k, q)
    finally:
        h.close()
