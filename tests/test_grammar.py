"""Connected words under a finite-state grammar (K6g, an extension the reference does not have; parity unpinned):
sr_connected_grammar_batch and sr_recognise_connected_grammar_batch.

CPU: the decoder's C restatement (tests/oracle_ext/long_grammar.c, capture form) equals gram_ref, a plain Python cell-level
reference written here from the definition in speech_recog.h, on random NFAs with segments; its totals equal a minimum
over accepted command sequences and segmentations built on the unnormalised full DTW of refs.py; the words are accepted,
tile every segment and carry their own path sums; the loop grammar is the K6 restatement; a chain of L states gives L words. GPU:
both calls equal the oracles bit for bit and write only their documented bytes; under the loop grammar they equal
sr_connected_batch and sr_recognise_connected_batch; a chain grammar recovers digit strings spoken across VAD pauses."""
import os

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import draw, make_slot, partition_grammar, random_bank, random_grammar
from drive import enrolled_bank, prefilled
from refs import MAX_A, MAX_B, NTHREADS, accepts, bank_members, copies_of, dtw_full, get_dis

P_MAX = 2 ** 32 - 1
PENALTIES = (0, 1, 1000, P_MAX)
TAG_MFCC, TAG_GRAM = 1, 10
INF64 = 2 ** 64 - 1
LOOP = sr_b200.loop_grammar()
NONE = ox.SEG_NONE


# ---- references ---------------------------------------------------------------------------------------------------
def _seg_of(seg, f):
    """(segment index, its first frame) of frame f"""
    g = max(k for k in range(3) if seg[k] != NONE and seg[k] <= f)
    return g, seg[g]


def gram_ref(x, bank, n_slot, grammar, P, seg=(0, NONE, NONE)):
    """the grammar decoder from its definition, cell by cell: (words [(slot, cmd, segment, start, end, dis)], total)"""
    S, F, _ = grammar
    N = len(x)
    if N == 0:
        return [], (0 if F & 1 else INF64)
    mem = bank_members(bank, n_slot, bank.shape[1])
    cps = copies_of(grammar, mem)
    inf = None
    D = [[inf] * len(mem[t]) for _, t, _ in cps]          # (D, start) of frame i-1; a cell key is (D, -start)
    E = []                                                # per frame: [(D, copy, start) or None] per state
    Eprev = [0] + [inf] * (S - 1)
    for i in range(N):
        if i in seg:
            D = [[inf] * len(r) for r in D]
        Ei = [inf] * S
        for c, (s, t, src) in enumerate(cps):
            y = mem[t]
            ein = [Eprev[q] for q in range(S) if src >> q & 1 and Eprev[q] is not inf]
            prev, row, diag = D[c], [], inf
            for j in range(len(y)):
                cands = [prev[j]]
                if j == 0:
                    cands += [(min(ein) + P, i)] if ein else []
                else:
                    cands += [row[j - 1], diag]
                diag = prev[j]
                cands = [q for q in cands if q is not inf]
                best = min(cands, key=lambda q: (q[0], -q[1])) if cands else inf
                row.append(inf if best is inf else (best[0] + get_dis(x[i], y[j]), best[1]))
            D[c] = row
            if row[-1] is not inf and (Ei[s] is inf or row[-1][0] < Ei[s][0]):
                Ei[s] = (row[-1][0], c, row[-1][1])
        E.append(Ei)
        Eprev = [e if e is inf else e[0] for e in Ei]
    fin = [s for s in range(S) if F >> s & 1 and E[-1][s] is not inf]
    if not fin:
        return [], INF64
    fs = min(fin, key=lambda s: (E[-1][s][0], s))
    words, i, s = [], N - 1, fs
    while i >= 0:
        d, c, b = E[i][s]
        prev = 0
        if b:
            src = cps[c][2]
            s = min((q for q in range(S) if src >> q & 1 and E[b - 1][q] is not inf), key=lambda q: (E[b - 1][q][0], q))
            prev = E[b - 1][s][0]
        g, f0 = _seg_of(seg, b)
        t = cps[c][1]
        words.append((t, t // 4, g, b - f0, i + 1 - f0, d - prev - P))
        i = b - 1
    return words[::-1], E[-1][fs][0]


def brute_total(x, mem, grammar, P, seg=(0, NONE, NONE)):
    """min over accepted command sequences and segmentations (no word crossing a segment boundary) of
    sum(dtw_full + P): a DP over (frame, state) built on whole-word DTWs"""
    S, F, arcs = grammar
    N = len(x)
    firsts = sorted(f for f in seg if f != NONE)
    seg_id = [max(k for k, f in enumerate(firsts) if f <= i) for i in range(N)]
    best = [[None] * S for _ in range(N + 1)]
    best[0][0] = 0
    for e in range(1, N + 1):
        for st in range(e):
            if seg_id[st] != seg_id[e - 1]:
                continue
            for s in range(S):
                if best[st][s] is None:
                    continue
                for t, y in mem.items():
                    cost = best[st][s] + dtw_full(x[st:e].astype(np.int64), y) + P
                    for a, b, m in arcs:
                        if a == s and (m >> (t // 4)) & 1 and (best[e][b] is None or cost < best[e][b]):
                            best[e][b] = cost
    fin = [best[N][s] for s in range(S) if F >> s & 1 and best[N][s] is not None]
    return min(fin) if fin else INF64


def _tuples(words, n):
    return [tuple(int(w[k]) for k in ("slot", "cmd", "segment", "start", "end", "dis")) for w in words[:n]]


def _random_segments(rng, N):
    """1-3 segments over N frames: the first frames (NONE where a segment has no frames)"""
    if N < 2:
        return (0, NONE, NONE)
    cuts = sorted(set(int(c) for c in rng.integers(1, N, int(rng.integers(0, 3)))))
    seg = [0] + cuts + [NONE] * (2 - len(cuts))
    if rng.random() < 0.2 and len(cuts) == 1:              # segment 1 empty, 2 with frames
        seg = [0, NONE, cuts[0]]
    return tuple(seg)


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_oracle_equals_cell_reference_and_brute_force():
    """sro_grammar == gram_ref on random NFAs of 1-5 states, random final masks, banks of 1-6 templates of 1-8 frames with
    erased, unsigned and frm_num 0 / 120 slots, N = 0..30 of tie-heavy {0, 1} and +-32 767 rows, every P, 1-3 segments;
    at N <= 8 the total equals brute_total (UINT64_MAX where nothing is accepted); the words' commands are accepted, the
    words tile every segment, each dis is the full DTW of its frames and sum(dis + P) = total"""
    go = ox.grammar()
    rng = np.random.default_rng(0x6A0)
    n_cases = n_multi = n_none = n_brute = 0
    for case in range(160):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = random_bank(rng, T, kind)
        g = random_grammar(rng)
        N = int(rng.integers(0, 31)) if case > 2 else case
        if case % 4 == 1:
            N = min(N, 8)
        x = draw(rng, N, kind)
        seg = _random_segments(rng, N)
        mem = bank_members(bank, T, bank.shape[1])
        for P in PENALTIES:
            feat = np.zeros((1, max(N, 1), 12), np.int16)
            feat[0, :N] = x
            w, nw, tot = go.decode(feat, [N], bank, T, bank.shape[1], g, P, 64, seg=[seg])
            want_words, want_total = gram_ref(x, bank, T, g, P, seg)
            got = _tuples(w[0], int(nw[0]))
            assert (got, int(tot[0])) == (want_words, want_total), (case, P)
            if 0 < N <= 8:
                assert want_total == brute_total(x, mem, g, P, seg), (case, P)
                n_brute += 1
            if not got:
                n_none += N > 0
                continue
            assert accepts(g, [c for _, c, _, _, _, _ in got]), (case, P)
            firsts = [f for f in seg if f != NONE]
            for k, f in enumerate(seg):
                if f == NONE:
                    continue
                ln = min([q for q in firsts if q > f] + [N]) - f
                ws = [q for q in got if q[2] == k]
                assert [q[3] for q in ws] == [0] + [q[4] for q in ws[:-1]] and ws[-1][4] == ln, (case, P, k)
            assert sum(q[5] + P for q in got) == want_total
            for slot, cmd, k, st, en, dis in got:
                assert cmd == slot // 4 and dis == dtw_full(x[seg[k] + st:seg[k] + en].astype(np.int64), mem[slot])
            n_cases += 1
            n_multi += len(got) > 1
    assert n_cases > 200 and n_multi > 50 and n_none > 20 and n_brute > 60, (n_cases, n_multi, n_none, n_brute)


def test_loop_grammar_is_the_connected_decoder():
    """the one-state loop grammar equals sro_connected bit for bit (words, n_words, total) on one segment, and on 2-3
    segments equals sro_connected of each segment on its own, words joined in order, totals summed"""
    go, co = ox.grammar(), ox.connected()
    rng = np.random.default_rng(0x6A1)
    for case in range(80):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = random_bank(rng, T, kind)
        if case % 16 == 15:
            bank[:] = 0xFF
        N = int(rng.integers(0, 41))
        x = draw(rng, N, kind)
        feat = np.zeros((1, max(N, 1), 12), np.int16)
        feat[0, :N] = x
        for P in PENALTIES:
            a = go.decode(feat, [N], bank, T, bank.shape[1], LOOP, P, 64)
            b = co.connected(feat, [N], bank, T, bank.shape[1], P, 64)
            for p, q in zip(a, b):
                assert np.array_equal(p, q), (case, P)
            seg = _random_segments(rng, N)
            w, nw, tot = go.decode(feat, [N], bank, T, bank.shape[1], LOOP, P, 64, seg=[seg])
            words, total = [], 0
            firsts = [f for f in seg if f != NONE]
            for k, f in enumerate(seg):
                if f == NONE or N == 0:
                    continue
                e = min([q for q in firsts if q > f] + [N])
                ww, wn, wt = co.connected(feat[:, f:e], [e - f], bank, T, bank.shape[1], P, 64)
                words += [(s, c, k, st, en, d) for s, c, _, st, en, d in _tuples(ww[0], int(wn[0]))]
                total = min(total + int(wt[0]), INF64)
            assert (_tuples(w[0], int(nw[0])), int(tot[0])) == (words, total), (case, P, seg)


def test_chain_gives_exactly_L_words():
    """a chain of L + 1 states (arcs k -> k+1 over every command, final state L) gives exactly L words whenever a path
    exists (L <= N), none otherwise, and each word lands in the next state"""
    go = ox.grammar()
    rng = np.random.default_rng(0x6A2)
    n_path = 0
    for case in range(60):
        T = int(rng.integers(1, 7))
        bank = random_bank(rng, T, ("tie", "small")[case % 2], plant=False)
        L = int(rng.integers(1, 6))
        N = int(rng.integers(0, 16))
        x = draw(rng, N, "small")
        feat = np.zeros((1, max(N, 1), 12), np.int16)
        feat[0, :N] = x
        g = sr_b200.chain_grammar(L, 0xFFFFFFFF)
        for P in (0, 1000):
            w, nw, tot = go.decode(feat, [N], bank, T, bank.shape[1], g, P, 16)
            if N >= L:
                assert int(nw[0]) == L and int(tot[0]) < INF64, (case, P)
                n_path += 1
            else:
                assert int(nw[0]) == 0 and int(tot[0]) == INF64, (case, P)
    assert n_path > 40


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _check_grammar(h, go, feat, frm, bank, T, stride, g, P, max_words, prefill=0x5A, seg=None):
    """the GPU decoder against the oracle, outputs prefilled: records past n_words keep their bytes; two launches agree"""
    h.set_bank(bank, T, stride)
    w0 = np.frombuffer(bytes([prefill]) * (len(frm) * max_words * 24), ox.WORD_DTYPE).reshape(len(frm), max_words).copy()
    got = h.connected_grammar(feat, frm, g, P, max_words, words=w0.copy())
    again = h.connected_grammar(feat, frm, g, P, max_words, words=w0.copy())
    ww, wn, wt = go.decode(feat, frm, bank, T, stride, g, P, max_words, nthreads=NTHREADS)
    assert np.array_equal(got[1], wn) and np.array_equal(got[2], wt)
    for b in range(len(frm)):
        k = min(int(wn[b]), max_words)
        assert np.array_equal(got[0][b, :k], ww[b, :k]), b
        assert np.array_equal(got[0][b, k:], w0[b, k:]), b
    for a, b in zip(got, again):
        assert np.array_equal(a, b)
    return got


@pytest.mark.gpu
def test_grammar_equals_oracle_over_lengths_copies_and_states():
    """N in {0, 1, 2, 119, 120, 500, 818}, copy counts 1, 8, 9, 64, 127 and 128 (every cluster width 1..16 occurs across
    the cases), 1, 2, 5, 12 and 16 states, more states than warps in the cluster (1 copy under 16 states, 8 under 12: a
    warp records several states), max_words below and above the word counts; tag 10 only"""
    go = ox.grammar()
    h = sr_b200.Handle(0)
    h.timing_enable(256)
    rng = np.random.default_rng(0x6A3)
    Ns = [0, 1, 2, 119, 120, 500, 818]
    widths = set()
    for C, S in ((1, 1), (8, 2), (9, 5), (64, 12), (127, 16), (128, 16), (17, 5), (40, 2), (100, 12), (120, 1), (56, 16),
                 (25, 12), (90, 5), (72, 2), (112, 16), (80, 1), (44, 12), (88, 5), (1, 16), (8, 12)):
        bank = random_bank(rng, 128, "small", stride=4096, fmin=1, fmax=119, plant=False)
        bank[rng.choice(128, 128 - C, replace=False)] = 0xFF
        g = partition_grammar(rng, S)
        assert len(copies_of(g, bank_members(bank, 128, 4096))) == C
        widths.add((C + 7) // 8)
        feat = np.zeros((len(Ns), 818, 12), np.int16)
        for k, N in enumerate(Ns):
            feat[k, :N] = draw(rng, N, "small")
        for P in ((0, 5000) if C < 64 else (3000,)):
            got = _check_grammar(h, go, feat, np.array(Ns, np.uint32), bank, 128, 4096, g, P, 6)
            assert got[1][0] == 0
        assert {t for t, _ in h.timing_collect()} == {TAG_GRAM}
    assert widths == set(range(1, 17))
    h.close()


@pytest.mark.gpu
def test_grammar_ties_headroom_averaged_bank_and_batch_position():
    """all-equal rows; the largest local distance at N = 818 (totals beyond 32 bits); random NFAs on tie-heavy rows; an
    sr_average_bank bank under the PIN and command-digit grammars; batch sizes around one and two passes of 132 clusters"""
    go = ox.grammar()
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0x6A4)
    eq = random_bank(rng, 24, "equal", stride=4096, fmin=1, fmax=119)
    feat = np.zeros((6, 818, 12), np.int16)
    feat[:] = draw(rng, 1, "equal")[0]
    frm = np.array([818, 1, 119, 300, 2, 817], np.uint32)
    for P in (0, 1, P_MAX):
        for g in (LOOP, sr_b200.chain_grammar(3, 0xFF), random_grammar(rng, 5)):
            _check_grammar(h, go, feat, frm, eq, 24, 4096, g, P, 900)
    big = np.stack([make_slot(np.tile(MAX_B, (119, 1)), 4096) for _ in range(40)])
    hf = np.tile(MAX_A, (4, 818, 1))
    got = _check_grammar(h, go, hf, np.full(4, 818, np.uint32), big, 40, 4096, sr_b200.chain_grammar(3, 0x3FF), P_MAX, 4)
    assert (got[2] > 2 ** 32).all() and (got[1] == 3).all()             # 3 x 40 = 120 copies
    _check_grammar(h, go, hf, np.full(4, 818, np.uint32), big, 40, 4096, LOOP, 0, 900)
    tie = random_bank(rng, 50, "tie", stride=4096, fmin=1, fmax=30)
    ft = np.stack([np.concatenate([draw(rng, 400, "tie"), np.zeros((418, 12), np.int16)]) for _ in range(5)])
    for P in (0, 1, 7):
        for S in (1, 2, 2):                                 # 50 slots: at most 2 states stay within 128 copies
            _check_grammar(h, go, ft, np.array([400, 399, 1, 37, 250], np.uint32), tie, 50, 4096, random_grammar(rng, S), P, 500)
    enr = h.enrol(sr_b200.synth_pcm_host(80, 8000, 0x6A40000), 2400)[0]
    avg = h.average_bank(enr, 4096, 4, 118, 2)[0]
    pcm = sr_b200.synth_pcm_host(16, 16000, 0x6A41000, 3)
    f, n = h.mfcc_long(pcm, np.array([[2400, 16000]] * 16, np.uint32), h.noise_atap(pcm, 2400), 818)
    pin = (5, 1 << 4, [(k, k + 1, 0x3FF) for k in range(4)])
    cmd_digit = (3, 1 << 2, [(0, 1, 0x3FC00), (1, 2, 0x3FF)])
    assert len(copies_of(pin, bank_members(avg, 80, 4096))) == 40
    for g in (pin, cmd_digit, LOOP):
        _check_grammar(h, go, f, n, avg, 80, 4096, g, 2000, 10)
    bank = random_bank(rng, 12, "small", stride=4096, fmin=2, fmax=40)
    g = random_grammar(rng, 4)
    lens = rng.integers(0, 160, 400).astype(np.uint32)
    feat = np.zeros((400, 160, 12), np.int16)
    for b in range(400):
        feat[b, :lens[b]] = draw(rng, int(lens[b]), "small")
    h.set_bank(bank, 12, 4096)
    ww, wn, wt = go.decode(feat, lens, bank, 12, 4096, g, 2500, 8, nthreads=NTHREADS)
    for lo, hi in ((0, 131), (131, 263), (0, 132), (5, 138), (100, 365), (0, 400), (399, 400)):
        got = h.connected_grammar(feat[lo:hi], lens[lo:hi], g, 2500, 8)
        assert np.array_equal(got[1], wn[lo:hi]) and np.array_equal(got[2], wt[lo:hi]), (lo, hi)
        for b in range(lo, hi):
            k = min(int(wn[b]), 8)
            assert np.array_equal(got[0][b - lo, :k], ww[b, :k])
    h.close()


@pytest.mark.gpu
def test_grammar_without_copies():
    """grammars with no copy against the bank -- the loop grammar on an erased and on an empty bank, arcs whose commands
    have no member, no arcs at all -- decode to 0 words with total 0 or UINT64_MAX as the definition says, at N = 0 and
    N > 0, equal to the oracle; on an erased bank the loop grammar still equals sr_connected_batch, at kernel level and
    end to end"""
    go = ox.grammar()
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0x6A9)
    Ns = np.array([0, 1, 5, 119, 818, 0], np.uint32)
    feat = np.zeros((len(Ns), 818, 12), np.int16)
    for k, N in enumerate(Ns):
        feat[k, :N] = draw(rng, int(N), "small")
    erased = np.full((12, 4096), 0xFF, np.uint8)
    digits = random_bank(rng, 12, "small", stride=4096, fmin=1, fmax=40, plant=False)   # commands 0..2 only
    empty = np.zeros((0, 4096), np.uint8)
    cases = [(erased, 12, LOOP), (empty, 0, LOOP), (digits, 12, (3, 1 << 2, [(0, 1, 1 << 20), (1, 2, 1 << 21)])),
             (digits, 12, (2, 1, [(0, 1, 0xFFFFFFF8)])), (digits, 12, (2, 3, [])), (digits, 12, (2, 2, []))]
    for bank, T, g in cases:
        assert not copies_of(g, bank_members(bank, T, 4096) if T else {})
        for P in (0, P_MAX):
            got = _check_grammar(h, go, feat, Ns, bank, T, 4096, g, P, 4)
            assert (got[1] == 0).all()
            assert list(got[2]) == [0 if N == 0 and g[1] & 1 else INF64 for N in Ns]
            if g is LOOP:                                   # word records: both calls leave them untouched
                want = h.connected(feat, Ns, P, 4)
                assert np.array_equal(want[1], got[1]) and np.array_equal(want[2], got[2]), (T, P)
    h.set_bank(erased, 12, 4096)
    pcm = sr_b200.synth_pcm_host(8, 16000, 0x6A91000, 3)
    for P in (0, 4000):
        a = h.recognise_connected(pcm, P, 4, out=prefilled(h, pcm, P, 4, 2400))
        b = h.recognise_connected_grammar(pcm, LOOP, P, 4, out=prefilled(h, pcm, P, 4, 2400))
        for k in a:
            assert np.array_equal(a[k], b[k]), (P, k)
        assert (b["n_words"] == 0).all() and (b["total"][b["frm_num"].sum(1) > 0] == INF64).all()
    h.close()


def _twin_case(rng):
    """a grammar whose trace-back meets a tie between source states: slots 0 (command 0) and 4 (command 1) hold the
    same template, reached through states 1 and 2, and both states lead to state 3 through slot 8 (command 2). E_1 = E_2
    at every frame, so the word before the last comes from state 1 -- slot 0 -- only because source ties go to the
    lowest state"""
    t, u = draw(rng, 6, "small"), draw(rng, 5, "small")
    bank = np.full((12, 4096), 0xFF, np.uint8)
    bank[0], bank[4], bank[8] = make_slot(t, 4096), make_slot(t, 4096), make_slot(u, 4096)
    g = (4, 1 << 3, [(0, 1, 1), (0, 2, 2), (1, 3, 4), (2, 3, 4)])
    feat = np.zeros((3, 40, 12), np.int16)
    frm = np.array([11, 40, 17], np.uint32)
    feat[0, :11] = np.concatenate([t, u])
    feat[1] = draw(rng, 40, "small")
    feat[2, :17] = np.concatenate([t, draw(rng, 3, "small"), u, draw(rng, 3, "small")])
    return bank, g, feat, frm


def test_source_ties_go_to_the_lowest_state():
    """on _twin_case the restatement equals gram_ref and traces the first word to slot 0"""
    go = ox.grammar()
    rng = np.random.default_rng(0x6AA)
    for case in range(8):
        bank, g, feat, frm = _twin_case(rng)
        for P in (0, 1000):
            w, nw, tot = go.decode(feat, frm, bank, 12, 4096, g, P, 4)
            for b in range(len(frm)):
                want = gram_ref(feat[b, :frm[b]], bank, 12, g, P)
                assert (_tuples(w[b], int(nw[b])), int(tot[b])) == want, (case, P, b)
                assert int(nw[b]) == 2 and [int(x) for x in w[b]["slot"][:2]] == [0, 8], (case, P, b)


@pytest.mark.gpu
def test_grammar_source_ties_on_gpu():
    """_twin_case on the GPU equals the restatement: the first word is slot 0"""
    go = ox.grammar()
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0x6AB)
    for case in range(8):
        bank, g, feat, frm = _twin_case(rng)
        for P in (0, 1000):
            got = _check_grammar(h, go, feat, frm, bank, 12, 4096, g, P, 4)
            assert (got[0][:, 0]["slot"] == 0).all(), (case, P)
    h.close()


@pytest.mark.gpu
def test_loop_grammar_equals_connected_batch():
    """the kernel-level loop grammar equals sr_connected_batch on random sequences against banks of 20 and 128 slots"""
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0x6A5)
    Ns = np.array([0, 1, 2, 118, 119, 120, 300, 818, 57, 3], np.uint32)
    feat = np.zeros((len(Ns), 818, 12), np.int16)
    for k, N in enumerate(Ns):
        feat[k, :N] = draw(rng, int(N), ("tie", "small")[k % 2])
    for T in (20, 128):
        h.set_bank(random_bank(rng, T, "small", stride=4096, fmin=1, fmax=119), T, 4096)
        for P in (0, 4000, P_MAX):
            a = h.connected(feat, Ns, P, 12)
            b = h.connected_grammar(feat, Ns, LOOP, P, 12)
            for p, q in zip(a, b):
                assert np.array_equal(p, q), (T, P)
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_loop_grammar_equals_recognise_connected(geom):
    """end to end, the loop grammar equals sr_recognise_connected_batch bit for bit (every output field, outputs
    prefilled) on the five board captures and synthetic captures at U = 8 000, 16 000 and 65 535"""
    h = sr_b200.Handle(0)
    h.set_geometry(geom)
    bank, _, _ = enrolled_bank(h, 20, 0x6A60000 + geom)
    h.set_bank(bank, 80, 4096)
    cap = np.load(os.path.join(os.path.dirname(__file__), "golden", "captures.npz"))
    cases = [np.stack([cap[k][:U] for k in sorted(cap.files) if len(cap[k]) >= U]) for U in (8000, 16000)]
    cases += [sr_b200.synth_pcm_host(B, U, 0x6A61000 + U, 3) for U, B in ((8000, 40), (16000, 40), (65535, 12))]
    for pcm in cases:
        for P, mw in ((0, 3), (4000, 8), (P_MAX, 2)):
            a = h.recognise_connected(pcm, P, mw, out=prefilled(h, pcm, P, mw, 2400))
            b = h.recognise_connected_grammar(pcm, LOOP, P, mw, out=prefilled(h, pcm, P, mw, 2400))
            for k in a:
                assert np.array_equal(a[k], b[k]), (pcm.shape, P, k)
    h.close()


def _paused_captures(h, ora, n_cmd, seed, n_cases, rng):
    """4 enrolled words, with pauses of 300 ms (the quiet tail of a capture) after some of them, so one string spans 2-3
    VAD segments; the later words at 85 % of their enrolled amplitude, so that no template matches exactly: (pcm
    [n_cases, U], command sequences, bank)"""
    bank, words_pcm, st = enrolled_bank(h, n_cmd, seed)
    atap = [ora.noise_atap(words_pcm[c], 2400) for c in range(n_cmd)]
    segs = [ora.vad(words_pcm[c], 8000, atap[c]).reshape(3, 2)[0] for c in range(n_cmd)]
    mid = [int(a["mid_val"][0]) for a in atap]
    U = 48000
    cands, seqs = [], []
    for case in range(n_cases):
        seq = [int(c) for c in rng.choice([c for c in range(n_cmd) if st[c] == 0], 4, replace=False)]
        lv = lambda c, y, a=1.0: np.clip(np.round((y.astype(np.int64) - mid[c]) * a).astype(np.int64) + mid[seq[0]], 0, 4095)
        tail = lv(seq[-1], words_pcm[seq[-1]][segs[seq[-1]][1]:])
        pause = np.tile(tail, 1 + 2400 // max(len(tail), 1))[:2400]
        gaps = [case % 3 == 0, case % 3 != 2, case % 3 == 2]      # one or two pauses after words 0, 1, 2
        parts = [words_pcm[seq[0]][:segs[seq[0]][1]]]
        for k, c in enumerate(seq[1:]):
            if gaps[k]:
                parts.append(pause)
            parts.append(lv(c, words_pcm[c][segs[c][0]:segs[c][1]], 0.85))
        x = np.concatenate(parts)
        x = np.concatenate([x, np.tile(tail, 1 + (U - len(x)) // max(len(tail), 1))])[:U]
        cands.append(x)
        seqs.append(seq)
    return np.stack(cands).astype(np.uint16), seqs, bank


@pytest.mark.gpu
def test_chain_grammar_recovers_strings_across_pauses():
    """4 words spliced with pauses longer than 110 ms, one string over 2-3 VAD segments: the call equals the composed
    oracle on every candidate (outputs prefilled); on the cases where the oracle recovers the spliced sequence, a 4-word
    chain grammar returns exactly that command sequence across segments"""
    go = ox.grammar()
    ora = ob.best_oracle()
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    n_cmd = 10
    rng = np.random.default_rng(0x6A7)
    pcm, seqs, bank = _paused_captures(h, ora, n_cmd, 0x6A70000, 24, rng)
    g = sr_b200.chain_grammar(4, (1 << n_cmd) - 1)
    want = ox.recognise_connected_grammar(ora, go, pcm, 2400, bank, 4 * n_cmd, 4096, g, 0, 8, nthreads=NTHREADS)
    nseg = (want["frm_num"] > 0).sum(1)
    keep = [b for b in range(len(seqs)) if want["status"][b] == 0 and nseg[b] >= 2
            and [int(w["cmd"]) for w in want["words"][b, :want["n_words"][b]]] == seqs[b]]
    assert len(keep) >= 3, len(keep)
    h.set_bank(bank, 4 * n_cmd, 4096)
    pre = prefilled(h, pcm, 0, 8, 2400)
    got = h.recognise_connected_grammar(pcm, g, 0, 8, out={k: v.copy() for k, v in pre.items()})
    for k in ("atap", "seg_off", "frm_num", "n_words", "total", "status"):
        assert np.array_equal(got[k], want[k]), k
    for b in range(len(seqs)):
        k = min(int(want["n_words"][b]), 8)
        assert np.array_equal(got["words"][b, :k], want["words"][b, :k]), b
        assert np.array_equal(got["words"][b, k:], pre["words"][b, k:]), b
    assert TAG_GRAM in {t for t, _ in h.timing_collect()}
    for b in keep:
        assert [int(w["cmd"]) for w in got["words"][b, :4]] == seqs[b]
        assert len(set(int(w["segment"]) for w in got["words"][b, :4])) >= 2
    h.close()


@pytest.mark.gpu
def test_grammar_argument_rules():
    """129 copies, 17 states, an arc to a state >= n_states, final_mask 0 or out of range, a NULL grammar and NULL arcs
    each fail, write nothing and launch nothing, in both calls; B = 0 launches nothing"""
    import ctypes as C
    h = sr_b200.Handle(0)
    L = sr_b200.lib()
    rng = np.random.default_rng(0x6A8)
    bank = random_bank(rng, 128, "small", stride=4096, fmin=2, fmax=40, plant=False)
    bank[1:4] = 0xFF                                        # 125 members: command 0 has one, command 1 four
    h.set_bank(bank, 128, 4096)
    one = (2, 2, [(0, 1, 1)])                               # 1 copy
    null_arcs = sr_b200.Grammar(2, 2, 1, C.cast(None, C.POINTER(sr_b200.GramArc)))
    assert len(copies_of((2, 2, [(0, 1, 0xFFFFFFFF), (1, 0, 2)]), bank_members(bank, 128, 4096))) == 129
    assert len(copies_of((2, 2, [(0, 1, 0xFFFFFFFF), (1, 0, 1), (0, 0, 4)]), bank_members(bank, 128, 4096))) == 130
    bad = [(2, 2, [(0, 1, 0xFFFFFFFF), (1, 0, 2)]),          # 125 + 4 = 129 copies
           (2, 2, [(0, 1, 0xFFFFFFFF), (1, 0, 1), (0, 0, 4)]),   # 130 copies
           (17, 1, [(0, 1, 1)]), (0, 1, []), (2, 2, [(0, 2, 1)]), (2, 2, [(2, 1, 1)]), (2, 0, [(0, 1, 1)]),
           (2, 4, [(0, 1, 1)]), None, null_arcs]
    lens = np.array([30, 0, 5, 12], np.uint32)
    f = np.zeros((4, 40, 12), np.int16)
    f[:] = draw(rng, 40, "small")
    pcm = sr_b200.synth_pcm_host(4, 8000, 0x6A80000, 3)
    for g in bad:
        gg = sr_b200.grammar(g)
        wbuf = np.full(4 * 3 * 24, 0x77, np.uint8)
        nw, tot = np.full(4, 0x77777777, np.uint32), np.full(4, 0x77, np.uint64)
        l0 = h.launch_count()
        rc = L.sr_connected_grammar_batch(h._h, sr_b200._p(f), sr_b200._p(lens), 40, 4, None if gg is None else C.byref(gg),
                                          5, 3, sr_b200._p(wbuf), sr_b200._p(nw), sr_b200._p(tot))
        assert rc != 0 and h.launch_count() == l0, g
        assert (wbuf == 0x77).all() and (nw == 0x77777777).all() and (tot == 0x77).all()
        out = {k: np.frombuffer(b"\x77" * v.nbytes, v.dtype).reshape(v.shape).copy()
               for k, v in h.recognise_connected(pcm[:1], 5, 3).items()}
        out = {k: np.repeat(v, 4, axis=0) for k, v in out.items()}
        pre = {k: v.copy() for k, v in out.items()}
        l0 = h.launch_count()
        with pytest.raises(sr_b200.SrError):
            h.recognise_connected_grammar(pcm, gg, 5, 3, out=out)
        assert h.launch_count() == l0, g
        for k in out:
            assert np.array_equal(out[k], pre[k]), (g, k)
    h.connected_grammar(f, lens, one, 5, 3)                 # the same arguments with a good grammar pass
    l0 = h.launch_count()
    assert L.sr_connected_grammar_batch(h._h, None, None, 0, 0, C.byref(sr_b200.grammar(one)), 0, 0, None, None, None) == 0
    o = sr_b200.ConnOut()
    assert L.sr_recognise_connected_grammar_batch(h._h, None, 0, 0, 0, C.byref(sr_b200.grammar(one)), 0, 0, C.byref(o)) == 0
    assert h.launch_count() == l0
    h.close()
