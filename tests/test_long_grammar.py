"""One grammar decode per long recording (K13, include/sr_long_grammar.h; an extension the reference does not have, parity
unpinned): sr_connected_grammar_segs_batch and sr_recognise_long_grammar_batch.

CPU: the decoder's C restatement (tests/oracle_ext/long_grammar.c) equals long_gram_ref, a plain Python cell-level reference
written here from the header's definition, on random NFAs over 1-40 segments with 0-frame segments interleaved; its words
are accepted, stay inside one segment, tile every decodable segment and sum with the penalties to the total; on <= 3
segments it is the capture decoder's restatement (sro_grammar_batch) and under the loop grammar the per-segment connected
decoder (sro_connected), joined. GPU: both calls equal the oracles bit for bit, including the u64 headroom corner, launch
cuts, threads and real speech; the loop grammar equals sr_connected_batch per segment and short recordings equal
sr_recognise_connected_grammar_batch."""
import os
import re
import threading

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from test_connected import _bank, _draw, _members, _slot
from test_grammar import accepts, copies_of, random_grammar
from test_long import FIXTURES, _bank_of, _synth_long
from test_long_edges import plant, plant_atap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P_MAX = 2 ** 32 - 1
PENALTIES = (0, 1, 1000, P_MAX)
INF64 = 2 ** 64 - 1
NULL = 0xFFFFFFFF
LOOP = sr_b200.loop_grammar()
TAG_MFCC, TAG_BLOCKS, TAG_SEGS, TAG_LONG_GRAM = 1, 11, 12, 13
REC_BYTES = 256 << 20              # kLongGramRecBytes, csrc/sr_api.cu: records per decoder launch
GROUP_BYTES = 256 << 20            # kLongGroupBytes: PCM per staged group
F_MAX = 1677720                    # SR_LONG_GRAM_FRM_MAX


# ---- the reference ------------------------------------------------------------------------------------------------------
def _get_dis(a, b):
    s = sum((int(p) - int(q)) ** 2 for p, q in zip(a, b)) & 0xFFFFFFFF
    return int(np.sqrt(np.float32(s)))


def long_gram_ref(x, seg_frm, bank, n_slot, grammar, P):
    """the decoder from sr_long_grammar.h's definition, cell by cell, over x = the segments' rows back to back: (words
    [(slot, cmd, segment, start, end, dis)], total)"""
    S, F, _ = grammar
    N = int(sum(seg_frm))
    if N == 0:
        return [], (0 if F & 1 else INF64)
    mem = _members(bank, n_slot, bank.shape[1])
    cps = copies_of(grammar, mem)
    seg_of, first = [], []                                # per frame: its segment, the segment's first frame
    for k, n in enumerate(seg_frm):
        seg_of += [k] * int(n)
        first += [len(first)] * int(n) if n else []
    inf = None
    D = [[inf] * len(mem[t]) for _, t, _ in cps]
    E, Eprev = [], [0] + [inf] * (S - 1)
    for i in range(N):
        if first[i] == i:                                 # a decodable segment's first frame
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
                row.append(inf if best is inf else (best[0] + _get_dis(x[i], y[j]), best[1]))
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
        t = cps[c][1]
        words.append((t, t // 4, seg_of[b], b - first[b], i + 1 - first[b], d - prev - P))
        i = b - 1
    return words[::-1], E[-1][fs][0]


def _tuples(words, n):
    return [tuple(int(w[k]) for k in ("slot", "cmd", "segment", "start", "end", "dis")) for w in words[:n]]


def _random_segs(rng, n_max=40, f_max=12):
    """1-n_max segments of 0-f_max frames, 0-frame segments interleaved"""
    n = int(rng.integers(1, n_max + 1))
    return [0 if rng.random() < 0.3 else int(rng.integers(1, f_max + 1)) for _ in range(n)]


def _check_words(words, total, seg_frm, grammar, P):
    """accepted by the grammar, inside one segment, tiling every decodable segment, sum(dis + P) == total"""
    if total == INF64:
        assert not words
        return
    assert accepts(grammar, [w[1] for w in words])
    assert sum(w[5] + P for w in words) == total
    pos = {k: 0 for k, n in enumerate(seg_frm) if n}
    for w in words:
        k, st, en = w[2], w[3], w[4]
        assert seg_frm[k] and st == pos[k] and st < en <= seg_frm[k]
        pos[k] = en
    assert all(pos[k] == seg_frm[k] for k in pos)


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_oracle_equals_python_reference():
    """sro_long_grammar == long_gram_ref on random NFAs of 1-5 states, banks of 1-6 templates with non-members planted,
    1-40 segments of 0-12 frames, tie-heavy {0, 1} and +-32 767 rows, every P; the words are accepted, stay inside their
    segment, tile every decodable segment and sum with P to the total"""
    lg = ox.long_grammar()
    rng = np.random.default_rng(0x13A)
    n_multi = 0
    for case in range(90):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = _bank(rng, T, kind)
        g = random_grammar(rng)
        segs = _random_segs(rng, 40 if case % 5 == 0 else 12, 12 if case % 5 == 0 else 6)
        x = _draw(rng, sum(segs), kind)
        for P in PENALTIES:
            w, nw, tot = lg.decode_segs(x, [0, len(segs)], segs, bank, T, bank.shape[1], g, P, 600)
            want_words, want_total = long_gram_ref(x, segs, bank, T, g, P)
            got = _tuples(w[0], int(nw[0]))
            assert (got, int(tot[0])) == (want_words, want_total), (case, P, segs)
            _check_words(got, int(tot[0]), segs, g, P)
            n_multi += len({q[2] for q in got}) > 1
    assert n_multi > 50


def test_oracle_equals_capture_decoder_on_three_segments():
    """with <= 3 segments of <= 818 frames in all, sro_long_grammar equals sro_grammar_batch given the segments' first
    frames: the adapter's three-entry table"""
    lg, go = ox.long_grammar(), ox.grammar()
    rng = np.random.default_rng(0x13B)
    for case in range(60):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = _bank(rng, T, kind)
        g = random_grammar(rng)
        nseg = int(rng.integers(1, 4))
        segs = [int(rng.integers(0, 30)) for _ in range(nseg)]
        if case == 0:
            segs = [300, 0, 518]                           # 818 frames in all
        N = sum(segs)
        x = _draw(rng, N, kind)
        first, f = [], 0
        for n in segs:
            first.append(f if n else ox.SEG_NONE)
            f += n
        first += [ox.SEG_NONE] * (3 - nseg)
        feat = np.zeros((1, max(N, 1), 12), np.int16)
        feat[0, :N] = x
        for P in PENALTIES:
            a = lg.decode_segs(x, [0, nseg], segs, bank, T, bank.shape[1], g, P, 900)
            b = go.decode(feat, [N], bank, T, bank.shape[1], g, P, 900, seg=[first])
            assert _tuples(a[0][0], int(a[1][0])) == _tuples(b[0][0], int(b[1][0])) and a[2][0] == b[2][0], (case, P)


def test_loop_grammar_equals_connected_per_segment():
    """under the loop grammar sro_long_grammar is sro_connected of each decodable segment alone, joined in order (each
    word keeping its segment), the totals summed"""
    lg, co = ox.long_grammar(), ox.connected()
    rng = np.random.default_rng(0x13C)
    for case in range(40):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = _bank(rng, T, kind)
        if not _members(bank, T, bank.shape[1]):
            continue
        segs = _random_segs(rng, 20, 15)
        x = _draw(rng, sum(segs), kind)
        for P in PENALTIES:
            w, nw, tot = lg.decode_segs(x, [0, len(segs)], segs, bank, T, bank.shape[1], LOOP, P, 400)
            want, total, r = [], 0, 0
            for k, n in enumerate(segs):
                if not n:
                    continue
                cw, cn, ct = co.connected(x[None, r:r + n], [n], bank, T, bank.shape[1], P, n)
                want += [(q[0], q[1], k, q[3], q[4], q[5]) for q in _tuples(cw[0], int(cn[0]))]
                total += int(ct[0])
                r += n
            assert _tuples(w[0], int(nw[0])) == want and int(tot[0]) == (total if sum(segs) else 0), (case, P)


def test_every_long_grammar_entry_point_is_run_here():
    """every sr_* entry point of include/sr_long_grammar.h is exercised by GPU tests of this file"""
    hdr = open(os.path.join(ROOT, "include", "sr_long_grammar.h")).read()
    names = set(re.findall(r"\bint\s+(sr_\w+)\s*\(", hdr))
    assert names == {"sr_connected_grammar_segs_batch", "sr_recognise_long_grammar_batch"}
    src = open(os.path.abspath(__file__)).read()
    py = {"sr_connected_grammar_segs_batch": ".connected_grammar_segs(", "sr_recognise_long_grammar_batch": ".recognise_long_grammar("}
    for n in names:
        assert src.count(py[n]) >= 3, n


# ---- GPU: the kernel-level form ------------------------------------------------------------------------------------------
def _flat(rng, seqs, kind="small"):
    """sequences given as lists of segment frame counts -> (feat [rows, 12], seq_seg, seg_frm)"""
    seg_frm = [n for s in seqs for n in s]
    seq_seg = np.cumsum([0] + [len(s) for s in seqs]).astype(np.uint32)
    return _draw(rng, int(sum(seg_frm)), kind), seq_seg, np.array(seg_frm, np.uint32)


def _check_segs(h, lg, feat, seq_seg, seg_frm, bank, T, g, P, max_words, prefill=0x5A):
    """the kernel-level call against the oracle; records past n_words keep the prefill"""
    B = len(seq_seg) - 1
    words = np.frombuffer(bytes([prefill]) * (B * max_words * 24), sr_b200.WORD_DTYPE).copy().reshape(B, max_words)
    w, nw, tot = h.connected_grammar_segs(feat, seq_seg, seg_frm, g, P, max_words, words=words)
    ww, wn, wt = lg.decode_segs(feat, seq_seg, seg_frm, bank, T, bank.shape[1], g, P, max_words)
    assert nw.tolist() == wn.tolist() and tot.tolist() == wt.tolist()
    for b in range(B):
        m = min(int(wn[b]), max_words)
        assert w[b, :m].tobytes() == ww[b, :m].tobytes(), b
        assert set(w[b, m:].tobytes()) <= {prefill}, b
    return nw, tot


def _partition_grammar(S, T, rng):
    """S states over the 2 * S commands of T = 8 S slots: state s is entered by commands 2s and 2s + 1 only (so every slot
    gives exactly one copy, C = T), from itself, from state s - 1 and from state 0; a random final mask"""
    arcs = []
    for s in range(S):
        m = 3 << (2 * s)
        for a in sorted({s, (s - 1) % S, 0}):
            arcs.append((a, s, m))
    return (S, int(rng.integers(1, 2 ** S)), arcs)


@pytest.mark.gpu
def test_segs_every_cluster_width_and_state_count(handle):
    """copy counts covering every cluster width 1..16 (C = 8 w copies: w CTAs) at w states, sequences of 1 and 2
    segments of 0, 1, 119, 120 and 818 frames and sequences with no decodable frame or no segment, every P"""
    lg = ox.long_grammar()
    rng = np.random.default_rng(0x13D)
    for w in range(1, 17):
        T = 8 * w
        bank = _bank(rng, T, ("small", "tie", "full")[w % 3], plant=False)
        handle.set_bank(bank, T, bank.shape[1])
        g = _partition_grammar(w, T, rng)
        assert len(copies_of(g, _members(bank, T, bank.shape[1]))) == T
        seqs = [[int(rng.choice([0, 1, 119, 120, 7]))], [0, 0], [818], [1, 0, 120], [], [119, 0, 1]]
        feat, seq_seg, seg_frm = _flat(rng, seqs, ("small", "tie", "full")[w % 3])
        for P in (PENALTIES[w % 4], 1000):
            _check_segs(handle, lg, feat, seq_seg, seg_frm, bank, T, g, P, 64)


@pytest.mark.gpu
def test_segs_many_segments(handle):
    """sequences of 819, 10 000 and 100 000 segments of 0-12 frames beside ones of 1 and 2, under a random NFA and the
    loop grammar, with max_words below and above the word counts"""
    lg = ox.long_grammar()
    rng = np.random.default_rng(0x13E)
    bank = _bank(rng, 12, "small")
    handle.set_bank(bank, 12, bank.shape[1])
    seqs = [[5], [3, 0], [int(rng.integers(0, 13)) for _ in range(819)], [int(rng.integers(0, 13)) for _ in range(10000)],
            [int(rng.integers(0, 4)) for _ in range(100000)], [0] * 1000]
    feat, seq_seg, seg_frm = _flat(rng, seqs)
    for g in (LOOP, random_grammar(np.random.default_rng(5), 4), (3, 4, [(0, 1, 0xF), (1, 2, 0xF0), (2, 0, 0x7)])):
        for mw in (7, 70000):
            nw, tot = _check_segs(handle, lg, feat, seq_seg, seg_frm, bank, 12, g, 1000, mw)
        if g is LOOP:
            assert int(nw[4]) > 60000 and int(nw[5]) == 0 and int(tot[5]) == 0


@pytest.mark.gpu
def test_segs_headroom(handle):
    """one sequence of 1 677 720 one-frame segments at P = 2^32 - 1 against a 119-frame template at the largest get_dis
    (65 536) from every input row: every frame is a forced word of dis 119 * 65 536 and the total is near 2^52.7. The total,
    every word and the word count equal the oracle's; beyond that sequence's frame limit the call fails"""
    lg = ox.long_grammar()
    x = np.zeros(12, np.int16)
    x[0] = 32767
    y = np.zeros(12, np.int16)
    y[0], y[1] = -32768, 362                                  # 65535^2 + 362^2 = 2^32 - 27: sqrtf rounds to 65 536
    assert _get_dis(x, y) == 65536
    bank = np.stack([_slot(np.tile(y, (119, 1)), 2880)])
    handle.set_bank(bank, 1, 2880)
    feat = np.tile(x, (F_MAX, 1))
    seg_frm = np.ones(F_MAX, np.uint32)
    w, nw, tot = handle.connected_grammar_segs(feat, [0, F_MAX], seg_frm, LOOP, P_MAX, F_MAX)
    ww, wn, wt = lg.decode_segs(feat, [0, F_MAX], seg_frm, bank, 1, 2880, LOOP, P_MAX, F_MAX)
    assert int(nw[0]) == int(wn[0]) == F_MAX
    assert int(tot[0]) == int(wt[0]) == F_MAX * (119 * 65536 + P_MAX)
    assert int(tot[0]) > 2 ** 52.68
    assert w.tobytes() == ww.tobytes()
    assert (w["dis"] == 119 * 65536).all() and (w["segment"] == np.arange(F_MAX)).all()
    with pytest.raises(sr_b200.SrError):
        handle.connected_grammar_segs(np.tile(x, (F_MAX + 1, 1)), [0, F_MAX + 1], np.ones(F_MAX + 1, np.uint32), LOOP, 0, 1)


@pytest.mark.gpu
def test_segs_argument_rules(handle):
    """a segment over 818 frames, a decreasing seq_seg and a malformed grammar fail before anything is written"""
    rng = np.random.default_rng(0x13F)
    bank = _bank(rng, 4, "small", plant=False)
    handle.set_bank(bank, 4, bank.shape[1])
    feat = _draw(rng, 900, "small")
    words = np.full((1, 4), 7, sr_b200.WORD_DTYPE)
    for seq_seg, seg_frm, g in (([0, 1], [819], LOOP), ([0, 2, 1], [1, 1], LOOP), ([0, 1], [5], (0, 1, []))):
        with pytest.raises(sr_b200.SrError):
            handle.connected_grammar_segs(feat, seq_seg, seg_frm, g, 0, 4, words=words)
        assert (words["slot"] == 7).all()


@pytest.mark.gpu
def test_segs_loop_grammar_equals_connected_per_segment(handle):
    """property 1 on the GPU: under the loop grammar the kernel-level call equals sr_connected_batch on each decodable
    segment alone, joined in order, the totals summed"""
    rng = np.random.default_rng(0x140)
    bank = _bank(rng, 20, "small")
    handle.set_bank(bank, 20, bank.shape[1])
    seqs = [[int(rng.choice([0, 1, 30, 119, 200, 818])) for _ in range(int(rng.integers(1, 12)))] for _ in range(40)]
    feat, seq_seg, seg_frm = _flat(rng, seqs)
    w, nw, tot = handle.connected_grammar_segs(feat, seq_seg, seg_frm, LOOP, 1000, 4000)
    row = np.cumsum(np.r_[0, seg_frm]).astype(np.int64)
    dec = [(b, k - int(seq_seg[b]), int(row[k]), int(seg_frm[k])) for b in range(len(seqs))
           for k in range(int(seq_seg[b]), int(seq_seg[b + 1])) if seg_frm[k]]
    X = np.zeros((len(dec), 818, 12), np.int16)
    fr = np.zeros(len(dec), np.uint32)
    for q, (_, _, r, n) in enumerate(dec):
        X[q, :n], fr[q] = feat[r:r + n], n
    cw, cn, ct = handle.connected(X, fr, 1000, 818)
    for b in range(len(seqs)):
        want, total = [], 0
        for q, (bb, k, _, _) in enumerate(dec):
            if bb == b:
                want += [(t[0], t[1], k, t[3], t[4], t[5]) for t in _tuples(cw[q], int(cn[q]))]
                total += int(ct[q])
        assert _tuples(w[b], int(nw[b])) == want and int(tot[b]) == total, b


# ---- GPU: the end-to-end form ----------------------------------------------------------------------------------------------
def _cmp_e2e(got, want, max_segs, max_words, rows=None):
    rows = range(len(want["n_segs"])) if rows is None else rows
    for b in rows:
        assert got["atap"][b].tobytes() == want["atap"][b].tobytes(), b
        assert int(got["n_segs"][b]) == int(want["n_segs"][b]), b
        m = min(int(want["n_segs"][b]), max_segs)
        for k in ("seg_off", "frm_num", "seg_status"):
            assert got[k][b, :m].tobytes() == want[k][b, :m].tobytes(), (b, k)
        assert int(got["n_words"][b]) == int(want["n_words"][b]) and int(got["total"][b]) == int(want["total"][b]), b
        m = min(int(want["n_words"][b]), max_words)
        assert got["words"][b, :m].tobytes() == want["words"][b, :m].tobytes(), b


def _planted_batch():
    """planted-activity recordings under PLANT_ATAP: segments over 818 frames, short ones, an open last segment and
    recordings without segments (a closed segment spans >= 8 + 2 frames of samples, so VAD never closes a 0-frame one)"""
    acts = []
    for runs in ([(12, 1), (20, 0), (900, 1), (15, 0), (30, 1), (11, 0)], [(9, 1), (11, 0)] * 30 + [(50, 1)],
                 [(5, 0)], [(818 + 9, 1), (11, 0), (8, 1), (11, 0), (1000, 1)], [(40, 0)]):
        acts.append(np.concatenate([np.full(n, v, np.uint8) for n, v in runs]))
    U = max(80 * len(a) + 160 for a in acts)
    pcm = np.full((len(acts), U), 2048, np.uint16)
    lens = np.zeros(len(acts), np.uint32)
    for b, a in enumerate(acts):
        p = plant(a)
        pcm[b, :len(p)] = p
        lens[b] = len(p)
    return pcm, lens


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_recognise_long_grammar_equals_composed_oracle(handle, geom):
    """synthetic recordings of ragged lengths and planted-activity ones (segments over 818 frames, an open last segment),
    three grammars, max_segs 0, 1, below and above n_segs, max_words below and above the word counts, prefilled outputs:
    every record equals the composed oracle and nothing outside the declared records is written"""
    lo, port, lg = ox.long_oracle(), ob.port(), ox.long_grammar()
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    handle.set_geometry(geom)
    try:
        lens = np.array([160, 161, 30000, 65535, 200001, 240000], np.uint32)
        pcm = _synth_long(lens, 240000, 0x1300)
        pp, pl = _planted_batch()
        cases = [(pcm, lens, 2400, None), (pp, pl, 0, plant_atap(len(pl)))]
        grams = (LOOP, sr_b200.chain_grammar(4, 0x7), (2, 3, [(0, 1, 0x5), (1, 0, 0xA), (1, 1, 0x1)]))
        for ci, (x, ln, n_len, at) in enumerate(cases):
            for gi, g in enumerate(grams):
                want = ox.recognise_long_grammar(lo, port, lg, x, n_len, bank, T, 4096, g, 1000, 64, 256, ln, geom == 1,
                                                 None if at is None else at.copy())
                ns = int(want["n_segs"].max())
                for max_segs, max_words in ((64, 256), (0, 3), (1, 1), (max(ns - 2, 1), 0)):
                    B = len(ln)
                    out = {"atap": np.zeros(B, ob.ATAP_DTYPE) if at is None else at.copy(),
                           "n_segs": np.full(B, 0xA5A5A5A5, np.uint32),
                           "seg_off": np.full((B, max_segs, 2), 0xA5A5A5A5, np.uint32),
                           "frm_num": np.full((B, max_segs), 0xA5A5A5A5, np.uint32), "seg_status": np.full((B, max_segs), 0xA5, np.uint8),
                           "n_words": np.full(B, 0xA5A5A5A5, np.uint32),
                           "words": np.frombuffer(b"\xa5" * (B * max_words * 24), sr_b200.WORD_DTYPE).copy().reshape(B, max_words),
                           "total": np.full(B, 0xA5A5A5A5A5A5A5A5, np.uint64)}
                    got = handle.recognise_long_grammar(x, g, 1000, max_segs, max_words, n_len, ln, out=out)
                    _cmp_e2e(got, want, max_segs, max_words)
                    for b in range(B):
                        m = min(int(want["n_segs"][b]), max_segs)
                        assert set(got["seg_off"][b, m:].tobytes()) <= {0xA5} and set(got["seg_status"][b, m:].tobytes()) <= {0xA5}
                        assert set(got["frm_num"][b, m:].tobytes()) <= {0xA5}
                        assert set(got["words"][b, min(int(want["n_words"][b]), max_words):].tobytes()) <= {0xA5}
                if ci == 1 and gi == 0:
                    st = want["seg_status"]
                    assert (st == 2).any() and (st == 1).any() and (st == 0).any(), st
        with pytest.raises(sr_b200.SrError):                  # lens > U fails, as sr_vad_long_batch does
            handle.recognise_long_grammar(pcm, LOOP, 0, 4, 4, 2400, np.r_[lens[:-1], 240001].astype(np.uint32))
    finally:
        handle.set_geometry(0)


@pytest.mark.gpu
def test_short_recordings_equal_the_capture_call(handle):
    """property 2: recordings of <= 65 535 samples (lens = U) whose long-form VAD finds <= 3 segments decode exactly as
    sr_recognise_connected_grammar_batch: words, n_words, total, atap, seg_off and frm_num"""
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    pcm = np.concatenate([sr_b200.synth_pcm_host(24, 40000, 0x1310, 3), ox.synth_long(8, 40000, 0x1311)])
    pcm = np.ascontiguousarray(pcm[:, :40000])
    for g in (LOOP, sr_b200.chain_grammar(3, 0x7), (2, 3, [(0, 1, 0x5), (1, 0, 0xA), (1, 1, 0x1)])):
        got = handle.recognise_long_grammar(pcm, g, 1000, 8, 64)
        cap = handle.recognise_connected_grammar(pcm, g, 1000, 64)
        ok = got["n_segs"] <= 3
        assert ok.sum() >= 24
        for b in np.flatnonzero(ok):
            n = int(got["n_segs"][b])
            assert got["atap"][b].tobytes() == cap["atap"][b].tobytes()
            assert got["seg_off"][b, :n].tobytes() == cap["seg_off"][b, :n].tobytes()
            assert got["frm_num"][b, :n].tobytes() == cap["frm_num"][b, :n].tobytes()
            assert int(got["n_words"][b]) == int(cap["n_words"][b]) and int(got["total"][b]) == int(cap["total"][b])
            m = min(int(cap["n_words"][b]), 64)
            assert got["words"][b, :m].tobytes() == cap["words"][b, :m].tobytes(), b


# ---- GPU: launches, scale and threads ------------------------------------------------------------------------------------
def _tags(h):
    t = [tag for tag, _ in h.timing_collect()]
    return {k: t.count(k) for k in set(t)}


def _cuts(N, S):
    """the host's rule: consecutive sequences while their records (N * S * 12 B) fit REC_BYTES, a sequence whose records
    alone exceed it on its own"""
    cuts, rows = [0], 0
    for b, n in enumerate(N):
        if rows and (rows + n) * S * 12 > REC_BYTES:
            cuts.append(b)
            rows = 0
        rows += n
    return cuts + [len(N)]


@pytest.mark.gpu
def test_record_cuts_and_launch_counts(handle):
    """a batch whose records cut into >= 3 decoder launches and a sequence whose records alone exceed the cap: launches
    per tag follow the host's rule, restated here, every row equals the oracle's and the one-launch slices of the batch"""
    lg = ox.long_grammar()
    rng = np.random.default_rng(0x141)
    bank = _bank(rng, 16, "small", plant=False)
    handle.set_bank(bank, 16, bank.shape[1])
    S = 16
    g = (S, 0xFFFF, [(k, (k + 1) % S, 0x1) for k in range(S)])   # 16 states x 4 slots of command 0: 64 copies
    # records of S * 12 B per frame: 1 400 000 frames is 269 MB, past the cap alone; 600 000 frames is 115 MB
    N = [600000, 600000, 1400000, 600000, 3]
    seqs = [[818] * (n // 818) + [n % 818] for n in N]
    feat, seq_seg, seg_frm = _flat(rng, seqs)
    cuts = _cuts(N, S)
    assert len(cuts) - 1 >= 3 and [cuts[k + 1] - cuts[k] for k in range(len(cuts) - 1)].count(1) >= 1
    handle.timing_enable(64)
    handle.timing_collect()
    c0 = handle.launch_count()
    w, nw, tot = handle.connected_grammar_segs(feat, seq_seg, seg_frm, g, 1000, 16)
    assert handle.launch_count() - c0 == len(cuts) - 1
    assert _tags(handle) == {TAG_LONG_GRAM: len(cuts) - 1}
    ww, wn, wt = lg.decode_segs(feat, seq_seg, seg_frm, bank, 16, bank.shape[1], g, 1000, 16)
    assert nw.tolist() == wn.tolist() and tot.tolist() == wt.tolist() and w.tobytes() == ww.tobytes()
    row = np.cumsum(np.r_[0, seg_frm])
    for k in range(len(cuts) - 1):
        a, b = cuts[k], cuts[k + 1]
        s0, s1 = int(seq_seg[a]), int(seq_seg[b])
        part = handle.connected_grammar_segs(feat[row[s0]:row[s1]], seq_seg[a:b + 1] - s0, seg_frm[s0:s1], g, 1000, 16)
        assert part[0].tobytes() == w[a:b].tobytes() and part[1].tolist() == nw[a:b].tolist() and part[2].tolist() == tot[a:b].tolist()
    handle.timing_collect()


@pytest.mark.gpu
def test_groups_and_launches_of_the_end_to_end_call():
    """per group of <= 256 MB of PCM: 2 launches of tag 11, 1 of tag 12, get_mfcc launches of tag 1 (8 192 pieces each)
    and the decoder's cuts of tag 13; rows equal a call per group"""
    h = sr_b200.Handle(0)
    try:
        h.set_bank(*ox.synth_bank(), 4096)
        h.timing_enable(4096)
        U = 1 << 24
        lens = np.array([U, U - 7, 3 * 80000, U, 161, U, U - 1, U, 999999, U], np.uint32)
        pcm = _synth_long(lens, U, 0x1320)
        G = max(1, GROUP_BYTES // (2 * U))
        groups = -(-len(lens) // G)
        assert G == 8 and groups == 2
        c0 = h.launch_count()
        got = h.recognise_long_grammar(pcm, LOOP, 1000, 64, 64, 2400, lens)
        n = h.launch_count() - c0
        t = _tags(h)
        assert t[TAG_BLOCKS] == 2 * groups and t[TAG_SEGS] == groups and t[TAG_LONG_GRAM] == groups
        assert t[TAG_MFCC] >= groups and n == sum(t.values()) + t[TAG_MFCC]   # one untimed gather per get_mfcc launch
        for g0 in range(0, len(lens), G):
            part = h.recognise_long_grammar(pcm[g0:g0 + G], LOOP, 1000, 64, 64, 2400, lens[g0:g0 + G])
            for k in got:
                assert part[k].tobytes() == got[k][g0:g0 + G].tobytes(), k
        h.timing_collect()
    finally:
        h.close()


@pytest.mark.gpu
def test_one_recording_of_2_27_samples(handle):
    """one recording of 2^27 samples end to end under a random grammar: equal to the composed oracle"""
    lo, port, lg = ox.long_oracle(), ob.port(), ox.long_grammar()
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    pcm = ox.synth_long(1, 1 << 27, 0x1330)
    g = (3, 5, [(0, 1, 0x3), (1, 2, 0x7), (2, 0, 0x7), (1, 1, 0x8)])
    got = handle.recognise_long_grammar(pcm, g, 1000, 100000, 400000)
    want = ox.recognise_long_grammar(lo, port, lg, pcm, 2400, bank, T, 4096, g, 1000, 100000, 400000)
    assert int(want["n_segs"][0]) > 1000
    _cmp_e2e(got, want, 100000, 400000)


@pytest.mark.gpu
def test_threads_beside_a_recognise_long_handle():
    """two long-grammar handles and a sr_recognise_long_batch handle on one GPU in threads: every result equals the
    serial run"""
    lens = np.array([90000, 150000, 40000], np.uint32)
    pcm = _synth_long(lens, 150000, 0x1340)
    chain = sr_b200.chain_grammar(5, 0x7)

    def job_a(h):
        return h.recognise_long_grammar(pcm, LOOP, 1000, 32, 64, 2400, lens)

    def job_b(h):
        w, nw, tot = h.connected_grammar_segs(_draw(np.random.default_rng(1), 3000, "small"), [0, 3, 5],
                                              [818, 0, 500, 818, 864 - 818], chain, 7, 64)
        r = h.recognise_long_grammar(pcm, chain, 7, 32, 64, 2400, lens)
        return dict(w=w, nw=nw, tot=tot, **r)

    def job_c(h):
        return h.recognise_long_batch(pcm, 32, 2400, lens)

    jobs = [job_a, job_b, job_c]
    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        for h in handles:
            h.set_bank(*ox.synth_bank(), 4096)
        serial = [j(h) for j, h in zip(jobs, handles)]
        results = [[None] * 3 for _ in jobs]
        errors = []

        def run(i):
            try:
                for rep in range(3):
                    results[i][rep] = jobs[i](handles[i])
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
                    assert np.asarray(results[i][rep][k]).tobytes() == np.asarray(v).tobytes(), (jobs[i].__name__, k)
    finally:
        for h in handles:
            h.close()


# ---- GPU: real speech ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_real_speech_digit_strings():
    """enrol one digit recording's segments (template k in slot 4k) and decode the other under the loop grammar, a chain
    of "any digit" positions as long as the enrolled list and the ordered chain: GPU equals the oracle. The accuracy (words
    whose command is their position) is printed and recorded in DESIGN.md, not asserted"""
    lo, port, lg = ox.long_oracle(), ob.port(), ox.long_grammar()
    h = sr_b200.Handle(0)
    try:
        for a_name, b_name in ((FIXTURES[0], FIXTURES[1]), (FIXTURES[1], FIXTURES[0]), (FIXTURES[2], FIXTURES[3]),
                               (FIXTURES[3], FIXTURES[2])):
            a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
            h.set_bank(np.zeros((0, 4096), np.uint8), 0, 4096)
            ea = h.recognise_long_batch(a[None], 32, 2400)
            ma = int(ea["n_segs"][0])
            ftr = ox.ftr_of_segments(port, a[None], ea["atap"], [(0, int(s["start"]), int(s["end"]) if s["end"] != NULL
                                                                  else int(s["start"])) for s in ea["segs"][0, :ma]])
            bank, T = _bank_of(ftr)
            h.set_bank(bank, T, 4096)
            K = T // 4
            any_digit = (1 << K) - 1
            grams = {"loop": LOOP, "any-digit chain": sr_b200.chain_grammar(K, any_digit),
                     "ordered chain": (K + 1, 1 << K, [(k, k + 1, 1 << k) for k in range(K)])}
            for name, g in grams.items():
                if name == "any-digit chain" and K * K > sr_b200.GRAM_COPY_MAX:   # K positions x K templates: too many copies
                    with pytest.raises(sr_b200.SrError):
                        h.recognise_long_grammar(b[None], g, 1000, 32, 64)
                    print("%s -> %s, %s: %d copies > %d" % (a_name, b_name, name, K * K, sr_b200.GRAM_COPY_MAX))
                    continue
                got = h.recognise_long_grammar(b[None], g, 1000, 32, 64)
                want = ox.recognise_long_grammar(lo, port, lg, b[None], 2400, bank, T, 4096, g, 1000, 32, 64)
                _cmp_e2e(got, want, 32, 64)
                n = int(got["n_words"][0])
                cmds = got["words"][0, :n]["cmd"].tolist()
                right = sum(1 for k, c in enumerate(cmds) if c == k)
                print("%s -> %s, %s: %d words, %d/%d in position, cmds %s" % (a_name, b_name, name, n, right, K, cmds))
    finally:
        h.close()
