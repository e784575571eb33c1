"""Connected words (K6, an extension the reference does not have; the decoder's parity is unpinned, the long front end is
pinned to the reference piece by piece): sr_mfcc_long_batch, sr_connected_batch and sr_recognise_connected_batch.

CPU: the decoder's C restatement (tests/oracle_ext/connected.c) equals cell_ref, a plain Python cell-level reference written
here from the definition in speech_recog.h; its total equals a brute-force minimum over segmentations built on
dist_matrix and dtw_full (which share no code with either); the P = 2^32 - 1 and the concatenated-templates properties
hold; the piecewise long-feature oracle at frm_cap = 119 equals the oracle's get_mfcc. GPU: all three calls equal the
oracles bit for bit and write only their documented bytes."""
import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from test_extension_refs import MAX_A, MAX_B, MAX_FRM, NTHREADS, dist_matrix

P_MAX = 2 ** 32 - 1
PENALTIES = (0, 1, 1000, P_MAX)
TAG_MFCC, TAG_CONN = 1, 9
SAVE = sr_b200.SAVE_MASK


# ---- references ---------------------------------------------------------------------------------------------------
def _get_dis(a, b):
    """get_dis (DTW.C:45-62) of two rows: u32-wrapped sum of squares, float32 square root, truncated"""
    s = sum((int(p) - int(q)) ** 2 for p, q in zip(a, b)) & 0xFFFFFFFF
    return int(np.sqrt(np.float32(s)))


def _members(bank, n_slot, stride):
    """{slot: rows [M, 12]} of the members: save_sign == SR_SAVE_MASK and 1 <= frm_num <= 119"""
    out = {}
    for t in range(n_slot):
        sign, n = np.frombuffer(bank[t, :4].tobytes(), np.uint16)
        if sign == SAVE and 1 <= n <= MAX_FRM:
            out[t] = bank[t, 4:4 + 24 * int(n)].view(np.int16).reshape(int(n), 12).astype(np.int64)
    return out


def cell_ref(x, bank, n_slot, stride, P):
    """the decoder from its definition, cell by cell: (words [(slot, cmd, start, end, dis)], total)"""
    N = len(x)
    if N == 0:
        return [], 0
    mem = _members(bank, n_slot, stride)
    if not mem:
        return [], 2 ** 64 - 1
    inf = None
    D = {t: [inf] * len(y) for t, y in mem.items()}      # (D, start) of frame i-1; a cell key is (D, -start)
    E = []                                                # (D, slot, start) per frame
    Eprev = 0
    for i in range(N):
        for t, y in mem.items():
            prev, row, diag = D[t], [], inf
            for j in range(len(y)):
                cands = [prev[j]]
                if j == 0:
                    cands.append((Eprev + P, i))
                else:
                    cands += [row[j - 1], diag]
                diag = prev[j]
                cands = [c for c in cands if c is not inf]
                best = min(cands, key=lambda c: (c[0], -c[1])) if cands else inf
                row.append(inf if best is inf else (best[0] + _get_dis(x[i], y[j]), best[1]))
            D[t] = row
        ends = [(D[t][-1][0], t, D[t][-1][1]) for t in mem if D[t][-1] is not inf]
        E.append(min(ends, key=lambda e: (e[0], e[1])))
        Eprev = E[-1][0]
    words, i = [], N - 1
    while i >= 0:
        d, t, st = E[i]
        prev = E[st - 1][0] if st else 0
        words.append((t, t // 4, st, i + 1, d - prev - P))
        i = st - 1
    return words[::-1], E[-1][0]


def dtw_full(a, b):
    """unnormalised DTW over the full matrix, no 2:1 guard: D(I-1, M-1)"""
    d = dist_matrix(a, b)
    I, M = d.shape
    D = np.zeros((I, M), np.int64)
    for i in range(I):
        for j in range(M):
            prev = [D[i - 1, j]] if i else []
            prev += [D[i, j - 1]] if j else []
            prev += [D[i - 1, j - 1]] if i and j else []
            D[i, j] = d[i, j] + (min(prev) if prev else 0)
    return int(D[I - 1, M - 1])


def brute_total(x, mem, P):
    """min over segmentations 0 = b_0 < ... < b_K = N and words t_k of sum(dtw_full(x[b_k-1:b_k], y_t_k) + P)"""
    N = len(x)
    best = [0] + [None] * N
    for e in range(1, N + 1):
        best[e] = min(best[s] + dtw_full(x[s:e], y) + P for s in range(e) for y in mem.values())
    return best[N]


# ---- inputs -------------------------------------------------------------------------------------------------------
def _slot(rows, stride, sign=SAVE, frm=None):
    s = np.full(stride, 0xFF, np.uint8)
    n = len(rows) if frm is None else frm
    s[:4] = np.frombuffer(np.array([sign, n], np.uint16).tobytes(), np.uint8)
    s[4:4 + rows.size * 2] = np.frombuffer(np.ascontiguousarray(rows, np.int16).tobytes(), np.uint8)
    return s


def _draw(rng, n, kind):
    if kind == "tie":                                     # rows from {0, 1}: ties everywhere
        return rng.integers(0, 2, (n, 12)).astype(np.int16)
    if kind == "full":                                    # +-32767
        return (rng.choice([-1, 1], (n, 12)) * 32767).astype(np.int16)
    if kind == "equal":
        return np.tile(np.array([7, -3, 11, 0, -25, 4, 9, -1, 2, 3, -8, 6], np.int16), (n, 1))
    return rng.integers(-3000, 3001, (n, 12)).astype(np.int16)


def _bank(rng, T, kind, stride=2880, fmin=1, fmax=8, plant=True):
    """T slots of fmin..fmax frames; with plant, non-members mixed in: erased, unsigned, frm_num 0 and frm_num 120"""
    bank = np.stack([_slot(_draw(rng, int(rng.integers(fmin, fmax + 1)), kind), stride) for _ in range(T)]) if T else \
        np.zeros((0, stride), np.uint8)
    if plant and T >= 3:
        for t in rng.choice(T, min(T - 1, max(1, T // 4)), replace=False):
            c = int(rng.integers(4))
            bank[t] = (np.full(stride, 0xFF, np.uint8) if c == 0 else _slot(_draw(rng, 3, kind), stride, sign=0) if c == 1
                       else _slot(np.zeros((0, 12)), stride, frm=0) if c == 2 else _slot(_draw(rng, 5, kind), stride, frm=120))
    return bank


def _as_tuples(words, n):
    return [(int(w["slot"]), int(w["cmd"]), int(w["start"]), int(w["end"]), int(w["dis"])) for w in words[:n]]


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_oracle_equals_cell_reference_and_brute_force():
    """sro_connected == cell_ref (n_words, words, total) on random banks of 1-6 templates of 1-8 frames with non-members
    planted, N = 0..40 of tie-heavy {0, 1} and +-32 767 rows, P in {0, 1, 1000, 2^32 - 1}, and an empty / all-non-member
    bank; the total equals brute_total, every word's dis equals dtw_full of its frames, the words tile [0, N) in order
    and sum(dis + P) = total"""
    co = ox.connected()
    rng = np.random.default_rng(0xC0)
    n_cases = n_multi = 0
    for case in range(96):
        kind = ("tie", "full", "small")[case % 3]
        T = int(rng.integers(1, 7))
        bank = _bank(rng, T, kind)
        if case % 16 == 15:
            bank[:] = 0xFF                                # no member at all
        N = int(rng.integers(0, 41)) if case > 2 else case
        x = _draw(rng, N, kind)
        mem = _members(bank, T, bank.shape[1])
        for P in PENALTIES:
            feat = np.zeros((1, max(N, 1), 12), np.int16)
            feat[0, :N] = x
            w, nw, tot = co.connected(feat, [N], bank, T, bank.shape[1], P, 64)
            want_words, want_total = cell_ref(x, bank, T, bank.shape[1], P)
            got = _as_tuples(w[0], int(nw[0]))
            assert (got, int(tot[0])) == (want_words, want_total), (case, P)
            assert (w[0][int(nw[0]):] == np.zeros(1, ox.WORD_DTYPE)).all()
            if N == 0 or not mem:
                assert got == [] and int(tot[0]) == (0 if N == 0 else 2 ** 64 - 1)
                continue
            if N <= 24 or P == 0:
                assert want_total == brute_total(x, mem, P), (case, P)
            assert [g[2] for g in got] == [0] + [g[3] for g in got[:-1]] and got[-1][3] == N
            assert sum(g[4] + P for g in got) == want_total
            for slot, cmd, st, en, dis in got:
                assert cmd == slot // 4 and dis == dtw_full(x[st:en].astype(np.int64), mem[slot])
            n_cases += 1
            n_multi += len(got) > 1
    assert n_cases > 250 and n_multi > 50


def test_max_penalty_gives_the_argmin_word():
    """P = 2^32 - 1: exactly one word, the argmin of the unnormalised full DTW, the lowest slot on a tie"""
    co = ox.connected()
    rng = np.random.default_rng(0xC1)
    for case in range(60):
        kind = ("tie", "small", "equal")[case % 3]
        T = int(rng.integers(1, 7))
        bank = _bank(rng, T, kind, fmax=10)
        mem = _members(bank, T, bank.shape[1])
        if not mem:
            continue
        N = int(rng.integers(1, 30))
        x = _draw(rng, N, kind)
        w, nw, tot = co.connected(x[None], [N], bank, T, bank.shape[1], P_MAX, 4)
        scores = {t: dtw_full(x.astype(np.int64), y) for t, y in mem.items()}
        best = min(scores, key=lambda t: (scores[t], t))
        assert int(nw[0]) == 1 and _as_tuples(w[0], 1) == [(best, best // 4, 0, N, scores[best])], case
        assert int(tot[0]) == scores[best] + P_MAX


def test_concatenated_templates_decode_back():
    """an input made of distinct templates back to back decodes, at P = 0, to total 0 and that sequence of slots"""
    co = ox.connected()
    rng = np.random.default_rng(0xC2)
    for case in range(40):
        T = int(rng.integers(2, 9))
        bank = np.stack([_slot(_draw(rng, int(rng.integers(2, 9)), "small"), 2880) for _ in range(T)])
        seq = rng.integers(0, T, int(rng.integers(1, 6)))
        parts = [bank[t, 4:4 + 24 * int(bank[t, 2:4].view(np.uint16)[0])].view(np.int16).reshape(-1, 12) for t in seq]
        x = np.concatenate(parts)
        w, nw, tot = co.connected(x[None], [len(x)], bank, T, 2880, 0, 8)
        assert int(tot[0]) == 0 and [int(s) for s in w[0]["slot"][:int(nw[0])]] == list(seq), case
        ends = np.cumsum([len(p) for p in parts])
        assert list(w[0]["end"][:len(seq)]) == list(ends) and (w[0]["dis"][:len(seq)] == 0).all()


def test_piecewise_long_features_at_119_equal_get_mfcc():
    """mfcc_long at frm_cap = 119 (one piece per segment) equals the oracle's get_mfcc on pinned rows, segments at sample 0,
    NULL and over-long ones included; and pieces at 120..239 frames are the frames of the shifted single pieces"""
    o = ob.port()
    rng = np.random.default_rng(0xC3)
    B, U = 24, 30000
    pcm = rng.integers(0, 4096, (B, U)).astype(np.uint16)
    atap = np.zeros(B, ob.ATAP_DTYPE)
    atap["mid_val"] = rng.integers(1800, 2300, B)
    st = rng.integers(0, 12000, B)
    st[:4] = 0
    en = st + 160 + 80 * rng.integers(-1, 240, B)
    seg = np.stack([st, en], 1).astype(np.uint32)
    seg[5] = ob.NULL
    feat, frm = ox.mfcc_long(o, pcm, seg, atap, 119)
    want = o.mfcc_batch(ob.pinned_rows(pcm, atap), np.where(seg == ob.NULL, ob.NULL, seg + 1), atap)
    assert np.array_equal(frm, want["frm_num"])
    for b in range(B):
        n = int(frm[b])
        assert np.array_equal(feat[b, :n].reshape(-1), want["mfcc_dat"][b][:n * 12])
    feat2, frm2 = ox.mfcc_long(o, pcm, seg, atap, 818)
    for b in range(B):
        n = int(frm2[b])
        if n > 119:                                     # frames 119.. = the segment that starts 80 * 119 samples later
            s2 = np.array([[seg[b, 0] + 80 * 119, seg[b, 1]]], np.uint32)
            f, k = ox.mfcc_long(o, pcm[b:b + 1], s2, atap[b:b + 1], 818)
            assert int(k[0]) == n - 119 and np.array_equal(feat2[b, 119:n], f[0, :n - 119])


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _segments(rng, U, frames, at0=2, nulls=1):
    """one segment per entry of `frames` (segments at sample 0 first), start random, end = start + 160 + 80 (F - 1) + slack"""
    seg = []
    for k, F in enumerate(frames):
        ln = min(160 + 80 * (F - 1) + int(rng.integers(0, 80)), U)
        s0 = 0 if k < at0 else int(rng.integers(0, U - ln + 1))
        seg.append((s0, min(s0 + ln, U)))
    seg = np.array(seg, np.uint32)
    seg[len(seg) - nulls:] = ob.NULL
    return seg


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_mfcc_long_equals_piecewise_oracle(geom):
    """sr_mfcc_long_batch == mfcc_long of the reference's own get_mfcc (the port for GEOM_B, its only checker) on segments
    of 1, 118-120, 237-239, 818 frames (and more than frm_cap), at sample 0, over full-range samples, with NULL segments;
    rows past frm_num keep the prefilled bytes; frm_cap = 119 equals sr_mfcc_batch; pieces are timed under tag 1"""
    o = ob.port() if geom else ob.best_oracle()
    rng = np.random.default_rng(0xC4 + geom)
    U = 65535
    frames = [1, 118, 119, 120, 237, 238, 239, 818, 500, 1, 300, 817, 2]
    B = len(frames)
    pcm = rng.integers(0, 65536, (B, U)).astype(np.uint16)
    pcm[1::2] &= 0x0FFF
    atap = np.zeros(B, ob.ATAP_DTYPE)
    atap["mid_val"] = rng.integers(1800, 2300, B)
    seg = _segments(rng, U, frames)
    h = sr_b200.Handle(0)
    h.set_geometry(geom)
    h.timing_enable(64)
    for cap in (818, 300, 119, 1):
        fill = np.full((B, cap, 12), -12345, np.int16)
        feat, frm = h.mfcc_long(pcm, seg, atap, cap, feat=fill.copy())
        want, wfrm = ox.mfcc_long(o, pcm, seg, atap, cap, geom_b=bool(geom))
        assert np.array_equal(frm, wfrm), cap
        for b in range(B):
            n = int(frm[b])
            assert np.array_equal(feat[b, :n], want[b, :n]), (cap, b)
            assert (feat[b, n:] == -12345).all(), (cap, b)
        assert {t for t, _ in h.timing_collect()} <= {TAG_MFCC}
        if cap == 119:
            f = h.mfcc(pcm, seg, atap)
            assert np.array_equal(f["frm_num"], frm)
            for b in range(B):
                assert np.array_equal(f["mfcc_dat"][b][:int(frm[b]) * 12], feat[b, :int(frm[b])].reshape(-1))
    assert (frm == 0).sum() >= 2
    with pytest.raises(sr_b200.SrError):
        h.mfcc_long(pcm, seg, atap, 819)
    with pytest.raises(sr_b200.SrError):
        h.mfcc_long(pcm, seg, atap, 0, feat=np.zeros((B, 0, 12), np.int16))
    h.close()


def _check_connected(h, co, feat, frm, bank, T, stride, P, max_words, prefill=0x5A):
    """the GPU decoder against the oracle, outputs prefilled: records past n_words keep their bytes; two launches agree"""
    h.set_bank(bank, T, stride)
    w0 = np.frombuffer(bytes([prefill]) * (len(frm) * max_words * 24), ox.WORD_DTYPE).reshape(len(frm), max_words).copy()
    got = h.connected(feat, frm, P, max_words, words=w0.copy())
    again = h.connected(feat, frm, P, max_words, words=w0.copy())
    ww, wn, wt = co.connected(feat, frm, bank, T, stride, P, max_words, nthreads=NTHREADS)
    assert np.array_equal(got[1], wn) and np.array_equal(got[2], wt)
    for b in range(len(frm)):
        k = min(int(wn[b]), max_words)
        assert np.array_equal(got[0][b, :k], ww[b, :k]), b
        assert np.array_equal(got[0][b, k:], w0[b, k:]), b
    for a, b in zip(got, again):
        assert np.array_equal(a, b)
    return got


@pytest.mark.gpu
def test_connected_equals_oracle_over_lengths_and_banks():
    """N in {0, 1, 2, 118, 119, 120, 237, 238, 500, 818} against banks of 1, 20, 32, 33, 80 and 128 (the limit) slots with
    non-members mixed in, every penalty, max_words smaller and larger than the word counts"""
    co = ox.connected()
    h = sr_b200.Handle(0)
    h.timing_enable(64)
    rng = np.random.default_rng(0xC5)
    Ns = [0, 1, 2, 118, 119, 120, 237, 238, 500, 818]
    for T in (1, 20, 32, 33, 80, 128):
        bank = _bank(rng, T, "small", stride=4096, fmin=1, fmax=119)
        feat = np.zeros((len(Ns), 818, 12), np.int16)
        for k, N in enumerate(Ns):
            feat[k, :N] = _draw(rng, N, "small")
        for P in ((0, 5000, P_MAX) if T < 80 else (3000,)):
            got = _check_connected(h, co, feat, np.array(Ns, np.uint32), bank, T, 4096, P, 6)
            assert (got[1][1:] >= 1).all() and got[1][0] == 0 and got[2][0] == 0
        assert {t for t, _ in h.timing_collect()} == {TAG_CONN}
    h.close()


@pytest.mark.gpu
def test_connected_ties_headroom_and_averaged_bank():
    """all-equal rows (every cell a tie); rows at the largest local distance at N = 818 against 119-frame templates (D
    beyond 32 bits); tie-heavy {0, 1} rows; a bank from sr_average_bank of enrolled groups"""
    co = ox.connected()
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0xC6)
    eq = _bank(rng, 24, "equal", stride=4096, fmin=1, fmax=119, plant=True)
    feat = np.zeros((6, 818, 12), np.int16)
    feat[:] = _draw(rng, 1, "equal")[0]
    frm = np.array([818, 1, 119, 300, 2, 817], np.uint32)
    for P in (0, 1, P_MAX):
        _check_connected(h, co, feat, frm, eq, 24, 4096, P, 900)
    big = np.stack([_slot(np.tile(MAX_B, (119, 1)), 4096) for _ in range(40)])
    hf = np.tile(MAX_A, (4, 818, 1))
    got = _check_connected(h, co, hf, np.full(4, 818, np.uint32), big, 40, 4096, P_MAX, 4)
    assert (got[2] > 2 ** 32).all()
    _check_connected(h, co, hf, np.full(4, 818, np.uint32), big, 40, 4096, 0, 900)
    tie = _bank(rng, 50, "tie", stride=4096, fmin=1, fmax=30)
    ft = np.stack([np.concatenate([_draw(rng, 400, "tie"), np.zeros((418, 12), np.int16)]) for _ in range(5)])
    for P in (0, 1, 7):
        _check_connected(h, co, ft, np.array([400, 399, 1, 37, 250], np.uint32), tie, 50, 4096, P, 500)
    enr = h.enrol(sr_b200.synth_pcm_host(80, 8000, 0xC60000), 2400)[0]
    avg = h.average_bank(enr, 4096, 4, 118, 2)[0]
    f, n = h.mfcc_long(sr_b200.synth_pcm_host(16, 16000, 0xC61000, 3), np.array([[2400, 16000]] * 16, np.uint32),
                       h.noise_atap(sr_b200.synth_pcm_host(16, 16000, 0xC61000, 3), 2400), 818)
    _check_connected(h, co, f, n, avg, 80, 4096, 2000, 10)
    h.close()


@pytest.mark.gpu
def test_connected_batch_position_and_argument_rules():
    """batch sizes around multiples of 132 and 264 clusters, every sequence equal to the oracle wherever it sits; an
    over-limit bank (129 slots), frm_num above 818 or frm_stride and a NULL n_words fail and write nothing; B = 0 launches
    nothing"""
    co = ox.connected()
    h = sr_b200.Handle(0)
    rng = np.random.default_rng(0xC7)
    bank = _bank(rng, 12, "small", stride=4096, fmin=2, fmax=40)
    lens = rng.integers(0, 160, 400).astype(np.uint32)
    feat = np.zeros((400, 160, 12), np.int16)
    for b in range(400):
        feat[b, :lens[b]] = _draw(rng, int(lens[b]), "small")
    h.set_bank(bank, 12, 4096)
    ww, wn, wt = co.connected(feat, lens, bank, 12, 4096, 2500, 8, nthreads=NTHREADS)
    for lo, hi in ((0, 131), (131, 263), (0, 132), (5, 138), (100, 365), (0, 400), (399, 400)):
        got = h.connected(feat[lo:hi], lens[lo:hi], 2500, 8)
        assert np.array_equal(got[1], wn[lo:hi]) and np.array_equal(got[2], wt[lo:hi]), (lo, hi)
        for b in range(lo, hi):
            k = min(int(wn[b]), 8)
            assert np.array_equal(got[0][b - lo, :k], ww[b, :k])
    wide = _bank(rng, 129, "small", stride=4096, fmin=2, fmax=40)
    L = sr_b200.lib()
    for bk, T, fr, stride, nw_null in ((wide, 129, lens[:4], 160, False), (bank, 12, np.array([819, 1, 1, 1], np.uint32), 900, False),
                                       (bank, 12, np.array([1, 161, 1, 1], np.uint32), 160, False), (bank, 12, lens[:4], 160, True)):
        h.set_bank(bk, T, 4096)
        f = np.zeros((4, stride, 12), np.int16)
        wbuf = np.full(4 * 3 * 24, 0x77, np.uint8)
        nw, tot = np.full(4, 0x77777777, np.uint32), np.full(4, 0x77, np.uint64)
        l0 = h.launch_count()
        rc = L.sr_connected_batch(h._h, sr_b200._p(f), sr_b200._p(np.ascontiguousarray(fr, np.uint32)), stride, 4, 5, 3,
                                  sr_b200._p(wbuf), None if nw_null else sr_b200._p(nw), sr_b200._p(tot))
        assert rc != 0 and h.launch_count() == l0
        assert (wbuf == 0x77).all() and (nw == 0x77777777).all() and (tot == 0x77).all()
    h.set_bank(bank, 12, 4096)
    l0 = h.launch_count()
    assert L.sr_connected_batch(h._h, None, None, 0, 0, 0, 0, None, None, None) == 0 and h.launch_count() == l0
    h.close()


def _check_recognise(h, co, pcm, bank, T, P, max_words, n_len=2400):
    """sr_recognise_connected_batch against the composed oracle, outputs prefilled with 0x5A: only the documented bytes change"""
    B = pcm.shape[0]
    h.set_bank(bank, T, 4096)
    out = {k: np.frombuffer(b"\x5a" * a.nbytes, a.dtype).reshape(a.shape).copy() for k, a in
           h.recognise_connected(pcm[:1], P, max_words, n_len).items()}
    out = {k: np.repeat(v, B, axis=0) for k, v in out.items()}
    pre = {k: v.copy() for k, v in out.items()}
    got = h.recognise_connected(pcm, P, max_words, n_len, out=out)
    want = ox.recognise_connected(ob.best_oracle(), co, pcm, n_len, bank, T, 4096, P, max_words, atap0=pre["atap"])
    for k in ("atap", "seg_off", "frm_num", "n_words", "total", "status"):
        assert np.array_equal(got[k], want[k]), k
    for b in range(B):
        k = min(int(want["n_words"][b]), max_words)
        assert np.array_equal(got["words"][b, :k], want["words"][b, :k]), b
        assert np.array_equal(got["words"][b, k:], pre["words"][b, k:]), b
    return got


def _enrolled_bank(h, n_cmd, seed):
    """one enrolled word per command at slot 4 * cmd (the other slots erased), from synthetic one-word captures"""
    pcm = sr_b200.synth_pcm_host(n_cmd, 8000, seed)
    enr, st = h.enrol(pcm, 2400)
    bank = np.full((4 * n_cmd, 4096), 0xFF, np.uint8)
    bank[::4] = enr
    return bank, pcm, st


@pytest.mark.gpu
def test_recognise_connected_equals_composed_oracle():
    """the five board captures and synthetic 3-word captures at U = 8 000, 16 000 and 65 535 against an enrolled bank"""
    import os
    co = ox.connected()
    h = sr_b200.Handle(0)
    bank, _, _ = _enrolled_bank(h, 20, 0xC80000)
    cap = np.load(os.path.join(os.path.dirname(__file__), "golden", "captures.npz"))
    for U in (8000, 16000):
        rows = [cap[k][:U] for k in sorted(cap.files) if len(cap[k]) >= U]
        got = _check_recognise(h, co, np.stack(rows), bank, 80, 4000, 6)
    for U, B in ((8000, 40), (16000, 40), (65535, 12)):
        pcm = sr_b200.synth_pcm_host(B, U, 0xC81000 + U, 3)
        for P, mw in ((0, 3), (4000, 8), (P_MAX, 2)):
            got = _check_recognise(h, co, pcm, bank, 80, P, mw)
        assert (got["status"] == 0).sum() > B // 2
    pcm = sr_b200.synth_pcm_host(9, 16000, 0xC82000, 3)
    _check_recognise(h, co, pcm, bank, 80, 100, 4, n_len=2399)     # atap untouched (n_len % 240 != 0)
    h.close()


@pytest.mark.gpu
def test_recognise_connected_decodes_spliced_words():
    """words spliced back to back with no pause form one segment of more than 119 frames: sr_recognise_batch reports
    SR_ST_MFCC_FAIL on it, the connected call returns the spliced command sequence. Frames that straddle a join match no
    template exactly, so the splices are chosen on the CPU first: only those from which the oracle recovers the sequence
    are kept, and the call must equal the oracle on every candidate"""
    co = ox.connected()
    ora = ob.best_oracle()
    h = sr_b200.Handle(0)
    n_cmd = 10
    bank, words_pcm, st = _enrolled_bank(h, n_cmd, 0xC90000)
    atap = [ora.noise_atap(words_pcm[c], 2400) for c in range(n_cmd)]
    segs = [ora.vad(words_pcm[c], 8000, atap[c]).reshape(3, 2)[0] for c in range(n_cmd)]
    mid = [int(a["mid_val"][0]) for a in atap]
    rng = np.random.default_rng(0xC9)
    U = 24000
    cands, seqs = [], []
    for _ in range(24):
        # four words (three are about 110 frames: too few), the later ones moved to the first capture's DC level
        seq = [int(c) for c in rng.choice([c for c in range(n_cmd) if st[c] == 0], 4, replace=False)]
        lv = lambda c, y: np.clip(y.astype(np.int64) - mid[c] + mid[seq[0]], 0, 4095)
        parts = [words_pcm[seq[0]][:segs[seq[0]][1]]] + [lv(c, words_pcm[c][segs[c][0]:segs[c][1]]) for c in seq[1:]]
        x = np.concatenate(parts)
        tail = lv(seq[-1], words_pcm[seq[-1]][segs[seq[-1]][1]:])
        x = np.concatenate([x, np.tile(tail, 1 + (U - len(x)) // max(len(tail), 1))])[:U]
        cands.append(x)
        seqs.append(seq)
    pcm = np.stack(cands).astype(np.uint16)
    want = ox.recognise_connected(ora, co, pcm, 2400, bank, 4 * n_cmd, 4096, 3000, 8)
    keep = [b for b in range(len(seqs)) if want["status"][b] == 0 and want["frm_num"][b, 0] > 119
            and [int(w["cmd"]) for w in want["words"][b, :want["n_words"][b]]] == seqs[b]]
    assert len(keep) >= 3, len(keep)
    got = _check_recognise(h, co, pcm, bank, 4 * n_cmd, 3000, 8)
    for b in keep:
        assert [int(w["cmd"]) for w in got["words"][b, :got["n_words"][b]]] == seqs[b]
        assert (got["words"][b, :4]["segment"] == 0).all()
    h.set_bank(bank, 4 * n_cmd, 4096)
    old = h.recognise(pcm[keep], 2400, want=("status",))
    assert (old["status"] == 2).all()
    h.close()
