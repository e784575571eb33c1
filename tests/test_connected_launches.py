"""The connected-word calls past their first launch. A large call is split three ways: get_mfcc pieces run kPieceChunk =
8 192 at a time (run_pieces: sr_mfcc_long_batch and both end-to-end calls), the grammar decoder's launches take
consecutive sequences whose records fit kGramRecBytes = 2^28 bytes (run_grammar), and every K6 / K6g launch takes at most
kSeqChunk = 2^20 sequences. Each later launch offsets its tables, features and outputs on its own, so an offset bug shows
only on the rows after the first launch.

Every case here: counts the launches under their timing tags (1 pieces, 9 K6, 10 K6g) against the plan the host uses, so
a changed constant fails loudly instead of silently no longer reaching the split; prefills the outputs (bytes past
n_words and rows past frm_num must survive); poisons the feature rows at and past frm_num with +-32 767; compares with the
oracle -- on the whole batch at kernel level, on the rows on both sides of every launch boundary plus the first, the
last and a few at random end to end -- and compares every row with the same call on slices that each make one launch."""
import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import draw, make_slot, partition_grammar, random_bank
from drive import enrolled_bank, prefilled
from refs import GRAM_REC_BYTES, NTHREADS, PIECE_CHUNK, SEQ_CHUNK, accepts, piece_plan, pieces, record_cuts, seq_launches

P_MAX = 2 ** 32 - 1
LOOP = sr_b200.loop_grammar()
TAG_MFCC, TAG_CONN, TAG_GRAM = 1, 9, 10
PREFILL = -12345
# poison for feature rows at and past frm_num: +-32 767 in a checkerboard over frames and coefficients
POISON = np.where((np.arange(818)[:, None] + np.arange(12)[None, :]) % 2, 32767, -32767).astype(np.int16)


# ---- plans: the host's splitting rules, restated in refs.py ------------------------------------------------------
def gram_launches(cuts):
    return len(seq_launches(cuts))


def _count(h, tag):
    return sum(1 for t, _ in h.timing_collect() if t == tag)


def _poisoned(rng, N, stride):
    """feature sequences of N[b] random rows, the rows at and past N[b] poisoned"""
    feat = rng.integers(-3000, 3001, (len(N), stride, 12), dtype=np.int16)
    past = np.arange(stride)[None, :] >= np.asarray(N, np.int64)[:, None]
    feat[past] = np.broadcast_to(POISON[:stride], feat.shape)[past]
    return feat


def _prefill_words(B, max_words):
    return np.frombuffer(b"\x5a" * (B * max_words * 24), ox.WORD_DTYPE).reshape(B, max_words).copy()


def _check_words(got, want, n_words, pre):
    """records below min(n_words, max_words) equal the oracle's, the rest keep the prefilled bytes"""
    B, mw = got.shape
    keep = np.arange(mw)[None, :] < np.minimum(n_words.astype(np.int64), mw)[:, None]
    g, w, p = (a.view(np.uint8).reshape(B, mw, 24) for a in (got, want, pre))
    bad = np.flatnonzero(~np.where(keep[:, :, None], g == w, g == p).all(axis=(1, 2)))
    assert bad.size == 0, "word records differ at sequences %s" % bad[:10].tolist()


def _equal_rows(a, b, what):
    bad = np.flatnonzero(~(a == b).reshape(len(a), -1).all(1)) if a.dtype.names is None else \
        np.flatnonzero(~(a.view(np.uint8).reshape(len(a), -1) == b.view(np.uint8).reshape(len(b), -1)).all(1))
    assert bad.size == 0, "%s differs at rows %s" % (what, bad[:10].tolist())


# ---- 1. sr_mfcc_long_batch across piece chunks --------------------------------------------------------------------
def _long_rows(rng, fmax):
    """(frames, at sample 0) per row, 0 frames for a NULL (-1) or short (-2) segment. At frm_cap = 818 the rows hold
    16 386+ pieces: launch 1 ends exactly between two segments, launch 2 ends inside a 7-piece segment at sample 0 (3 of
    its pieces in launch 2, 4 in launch 3), and launch 2 and the tail start with a segment at sample 0. Rows of 6 pieces
    (596..714 frames) outnumber those of 7 (715..818), so frm_cap = 714, where the 7-piece rows are over the cap, still
    makes two launches."""
    rows = [(1, True), (119, False), (120, True), (238, False), (239, True), (-1, False), (-2, False), (fmax, True),
            (714, False), (715, False), (1, False)]
    pat = (6, 7, 6, 6, 7)

    def piece_row(p, at0=False):
        rows.append((int(rng.integers(119 * (p - 1) + 1, min(119 * p, fmax) + 1)), at0))

    def fill_to(target):
        cum = int(pieces([max(F, 0) for F, _ in rows]).sum())
        while target - cum > 14:
            if rng.random() < 0.01:
                rows.append((int(rng.choice([-1, -2])), False))
            p = pat[len(rows) % 5]
            piece_row(p, rng.random() < 0.01)
            cum += p
        r = target - cum                                  # 8..14: one row of r - 7 pieces and one of 7
        piece_row(r - 7)
        piece_row(7)

    fill_to(PIECE_CHUNK)
    piece_row(6, True)                                    # launch 2's first piece pins x[-1]
    fill_to(2 * PIECE_CHUNK - 3)
    piece_row(7, True)                                    # pieces 16 381..16 387: the boundary falls inside
    rows += [(-1, False), (1, True), (600, False), (-2, False), (300, False), (fmax, False)]
    return rows


def _long_segments(rng, rows, U, frame_len):
    seg = np.zeros((len(rows), 2), np.uint32)
    for b, (F, at0) in enumerate(rows):
        if F == -1:
            seg[b] = ob.NULL
            continue
        ln = frame_len - 1 - int(rng.integers(0, 40)) if F == -2 else frame_len + 80 * (F - 1)
        ln = min(ln + (int(rng.integers(0, 80)) if F > 0 else 0), U)
        s0 = 0 if at0 else int(rng.integers(0, U - ln + 1))
        seg[b] = (s0, s0 + ln)
    return seg


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_mfcc_long_across_piece_chunks(geom):
    """sr_mfcc_long_batch at U = 65 535 on ~2 570 rows: at frm_cap = 818 three piece launches (one boundary between two
    segments, one inside a segment at sample 0), at frm_cap = 714 two (the 7-piece rows over the cap); NULL, short and
    sample-0 segments mixed in. The oracle (the port for GEOM_B) on the rows at every boundary, the first, the last and a
    few at random; row slices of one launch each equal the whole call on every row; rows past frm_num keep their bytes"""
    o = ob.port() if geom else ob.best_oracle()
    frame_len = 200 if geom else 160
    U = 65535
    fmax = (U - frame_len) // 80 + 1
    rng = np.random.default_rng(0xC1A0 + geom)
    rows = _long_rows(rng, fmax)
    B = len(rows)
    seg = _long_segments(rng, rows, U, frame_len)
    F = np.array([ox.long_frames(int(s), int(e), U, frame_len) for s, e in seg], np.int64)
    assert list(F) == [max(f, 0) for f, _ in rows]
    pcm = rng.integers(0, 65536, (B, U), dtype=np.uint16)
    pcm[1::2] &= 0x0FFF
    atap = np.zeros(B, ob.ATAP_DTYPE)
    atap["mid_val"] = rng.integers(1800, 2300, B)
    h = sr_b200.Handle(0)
    h.set_geometry(geom)
    h.timing_enable(64)
    for cap, want_launches in ((818, 3), (714, 2)):
        Fc = np.where(F <= cap, F, 0)
        launches, edge, slices = piece_plan(pieces(Fc))
        print("geom %d frm_cap %d: %d rows, %d pieces, %d launches, boundary rows %s, slices %s" % (
            geom, cap, B, int(pieces(Fc).sum()), launches, sorted(edge), slices))
        assert launches == want_launches
        fill = np.full((B, cap, 12), PREFILL, np.int16)
        feat, frm = h.mfcc_long(pcm, seg, atap, cap, feat=fill.copy())
        assert _count(h, TAG_MFCC) == launches
        assert np.array_equal(frm, Fc)
        past = np.arange(cap)[None, :] >= frm[:, None].astype(np.int64)
        assert (feat[past] == PREFILL).all()
        idx = sorted(edge | set(rng.choice(B, 4, replace=False).tolist()))
        want, wfrm = ox.mfcc_long(o, pcm[idx], seg[idx], atap[idx], cap, geom_b=bool(geom))
        assert np.array_equal(frm[idx], wfrm)
        for q, b in enumerate(idx):
            assert np.array_equal(feat[b, :frm[b]], want[q, :frm[b]]), (cap, b)
        for lo, hi in slices:
            f, n = h.mfcc_long(pcm[lo:hi], seg[lo:hi], atap[lo:hi], cap, feat=fill[lo:hi].copy())
            assert _count(h, TAG_MFCC) == 1, (cap, lo, hi)
            assert np.array_equal(n, frm[lo:hi])
            _equal_rows(f, feat[lo:hi], "features of slice %d..%d at frm_cap %d" % (lo, hi, cap))
    h.close()


# ---- 2. end to end across piece chunks ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_recognise_connected_across_piece_chunks():
    """4 400 synthetic 3-word captures at U = 16 000 (two launches of get_mfcc pieces) through sr_recognise_connected_batch
    and sr_recognise_connected_grammar_batch under the PIN chain and the loop grammar: the composed oracles on the
    captures at the piece boundary, the first and the last and a few at random; capture slices of one piece launch each
    equal the whole call on every capture; the loop grammar equals sr_recognise_connected_batch on the whole batch"""
    co, go, ora = ox.connected(), ox.grammar(), ob.best_oracle()
    h = sr_b200.Handle(0)
    bank, _, _ = enrolled_bank(h, 20, 0xC1B0000)
    h.set_bank(bank, 80, 4096)
    B, U, P, mw = 4400, 16000, 4000, 3
    pcm = sr_b200.synth_pcm_host(B, U, 0xC1B1000, 3)
    rng = np.random.default_rng(0xC1B)
    h.timing_enable(64)
    calls = (("connected", None), ("pin", sr_b200.chain_grammar(4)), ("loop", LOOP))
    whole = {}
    for name, g in calls:
        out = prefilled(h, pcm, P, mw, 2400)
        pre = {k: v.copy() for k, v in out.items()}
        run = (lambda x, o: h.recognise_connected(x, P, mw, out=o)) if g is None else \
            (lambda x, o, g=g: h.recognise_connected_grammar(x, g, P, mw, out=o))
        _count(h, TAG_MFCC)
        got = run(pcm, out)
        launches, edge, slices = piece_plan(pieces(got["frm_num"]).sum(1))
        print("%s: %d captures, %d pieces, %d launches, boundary captures %s, slices %s" % (
            name, B, int(pieces(got["frm_num"]).sum()), launches, sorted(edge), slices))
        assert launches >= 2 and _count(h, TAG_MFCC) == launches
        idx = sorted(edge | set(rng.choice(B, 3, replace=False).tolist()))
        if g is None:
            want = ox.recognise_connected(ora, co, pcm[idx], 2400, bank, 80, 4096, P, mw, atap0=pre["atap"][idx])
        else:
            want = ox.recognise_connected_grammar(ora, go, pcm[idx], 2400, bank, 80, 4096, g, P, mw,
                                                  atap0=pre["atap"][idx], nthreads=NTHREADS)
        for k in ("atap", "seg_off", "frm_num", "n_words", "total", "status"):
            assert np.array_equal(got[k][idx], want[k]), (name, k)
        _check_words(got["words"][idx], want["words"], want["n_words"], pre["words"][idx])
        for lo, hi in slices:
            o = {k: v[lo:hi].copy() for k, v in pre.items()}
            part = run(pcm[lo:hi], o)
            assert _count(h, TAG_MFCC) == 1, (name, lo, hi)
            for k in part:
                _equal_rows(part[k], got[k][lo:hi], "%s %s of slice %d..%d" % (name, k, lo, hi))
        whole[name] = got
    for k in whole["connected"]:
        _equal_rows(whole["loop"][k], whole["connected"][k], "loop grammar against K6: " + k)
    h.close()


# ---- 3. grammar record cuts at kernel level -----------------------------------------------------------------------
def _record_lengths(rng, S, n_launch):
    """sequence lengths for n_launch record launches at S states: zeros mixed in; at S = 16 launch 1 fills 2^28 bytes of
    records exactly (2^21 rows) and an N = 0 sequence after it stays in it; two N = 0 sequences end every launch"""
    limit = GRAM_REC_BYTES // (S * 8)
    draw = lambda: 0 if rng.random() < 0.03 else int(rng.integers(1, 300) if rng.random() < 0.1 else rng.integers(500, 819))
    N, rows = [], 0
    if S == 16:
        while rows + 818 <= limit - 818:
            N.append(draw())
            rows += N[-1]
        N += [limit - rows - 818, 818, 0]                # 818..1635 rows left: two sequences
        rows = limit
    while rows < (n_launch - 0.5) * limit:
        N.append(draw())
        rows += N[-1]
    cuts = record_cuts(N, S)
    for c in reversed(cuts[1:-1]):                       # zeros never cut: they stay at the end of the launch before
        N[c:c] = [0, 0]
    return np.array(N, np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("S", (16, 15))
def test_grammar_record_cuts(S):
    """sr_connected_grammar_batch over three record launches at 16 states (launch 1 exactly 2^28 bytes: 2^21 rows) and at
    15 (a row limit of 2 236 962, not a power of two) against 16 members of 1-8 frames, one per command; N = 0 sequences
    at every cut; max_words below (P = 0) and above (P = 2^32 - 1) the word counts. The oracle on the whole batch; slices
    of one launch each equal the whole call"""
    go = ox.grammar()
    rng = np.random.default_rng(0xC1C0 + S)
    bank = random_bank(rng, 64, "small", stride=4096, fmin=1, fmax=8, plant=False)
    bank[np.arange(64) % 4 != 0] = 0xFF                   # slot 4c holds command c's one member
    g = partition_grammar(rng, S, n_cmd=16)
    N = _record_lengths(rng, S, 3)
    cuts = record_cuts(N, S)
    rows = [int(N[lo:hi].sum()) for lo, hi in zip(cuts[:-1], cuts[1:])]
    print("S %d: %d sequences, record launches at %s, rows %s (limit %d)" % (S, len(N), cuts, rows, GRAM_REC_BYTES // (S * 8)))
    assert len(cuts) - 1 == 3 and all(N[c - 1] == 0 for c in cuts[1:-1])
    if S == 16:
        assert rows[0] == 1 << 21 and N[cuts[1] - 1] == 0
    feat = _poisoned(rng, N, 818)
    h = sr_b200.Handle(0)
    h.set_bank(bank, 64, 4096)
    h.timing_enable(64)
    for P, mw in ((0, 3), (P_MAX, 3)):
        ww, wn, wt = go.decode(feat, N, bank, 64, 4096, g, P, mw, nthreads=NTHREADS)
        w0 = _prefill_words(len(N), mw)
        got = h.connected_grammar(feat, N, g, P, mw, words=w0.copy())
        assert _count(h, TAG_GRAM) == gram_launches(cuts) == 3
        assert np.array_equal(got[1], wn) and np.array_equal(got[2], wt), P
        _check_words(got[0], ww, wn, w0)
        if P == 0:
            assert (wn > mw).mean() > 0.5
        else:
            assert ((wn > 0) & (wn < mw)).mean() > 0.5
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            part = h.connected_grammar(feat[lo:hi], N[lo:hi], g, P, mw, words=w0[lo:hi].copy())
            assert _count(h, TAG_GRAM) == 1, (P, lo, hi)
            for a, b in zip(part, got):
                _equal_rows(a, b[lo:hi], "slice %d..%d at P %d" % (lo, hi, P))
    h.close()


# ---- 4. more than 2^20 sequences in one call ----------------------------------------------------------------------
def _many_short(rng):
    """2^20 + 5 sequences of 0..2 frames (stride 2) against 13 slots (a 2-CTA cluster; non-members mixed in) in which
    slots 1 and 6 hold distinct 1-frame templates; the sequences at 2^20 - 1, 2^20, 2^20 + 1 and B - 1 are those two
    templates back to back"""
    B = SEQ_CHUNK + 5
    bank = random_bank(rng, 13, "small", stride=4096, fmin=1, fmax=3)
    ya, yb = draw(rng, 1, "small"), draw(rng, 1, "small")
    bank[1], bank[6] = make_slot(ya, 4096), make_slot(yb, 4096)
    N = rng.integers(0, 3, B).astype(np.uint32)
    plant = [SEQ_CHUNK - 1, SEQ_CHUNK, SEQ_CHUNK + 1, B - 1]
    N[plant] = 2
    feat = _poisoned(rng, N, 2)
    feat[plant] = np.concatenate([ya, yb])
    return B, bank, N, feat, plant


def _check_plants(got, plant, mw):
    for b in plant:
        assert int(got[1][b]) == 2 and int(got[2][b]) == 0, b
        assert [tuple(int(got[0][b, k][f]) for f in ("slot", "start", "end", "dis")) for k in range(2)] == \
            [(1, 0, 1, 0), (6, 1, 2, 0)], b


@pytest.mark.gpu
def test_connected_over_2_20_sequences():
    """sr_connected_batch on 2^20 + 5 sequences: two K6 launches; the whole batch equals the oracle, the planted
    sequences on both sides of the split decode to slots 1 then 6 at P = 0; [0, 2^20) and [2^20, B) alone equal it"""
    co = ox.connected()
    rng = np.random.default_rng(0xC1D)
    B, bank, N, feat, plant = _many_short(rng)
    h = sr_b200.Handle(0)
    h.set_bank(bank, 13, 4096)
    h.timing_enable(64)
    mw = 3
    w0 = _prefill_words(B, mw)
    got = h.connected(feat, N, 0, mw, words=w0.copy())
    assert _count(h, TAG_CONN) == 2
    ww, wn, wt = co.connected(feat, N, bank, 13, 4096, 0, mw, nthreads=NTHREADS)
    assert np.array_equal(got[1], wn) and np.array_equal(got[2], wt)
    _check_words(got[0], ww, wn, w0)
    _check_plants(got, plant, mw)
    for lo, hi in ((0, SEQ_CHUNK), (SEQ_CHUNK, B)):
        part = h.connected(feat[lo:hi], N[lo:hi], 0, mw, words=w0[lo:hi].copy())
        assert _count(h, TAG_CONN) == 1
        for a, b in zip(part, got):
            _equal_rows(a, b[lo:hi], "slice %d..%d" % (lo, hi))
    h.close()


@pytest.mark.gpu
def test_grammar_over_2_20_sequences():
    """sr_connected_grammar_batch on the same 2^20 + 5 sequences under an 8-state grammar that accepts the planted pair:
    the records fit one run_grammar launch, which makes two K6g launches; at 16 states and N = 2 everywhere the record
    cut falls at 2^20 itself (two launches again). The whole batch equals the oracle; slices of one launch equal it"""
    go = ox.grammar()
    rng = np.random.default_rng(0xC1E)
    B, bank, N, feat, plant = _many_short(rng)
    h = sr_b200.Handle(0)
    h.set_bank(bank, 13, 4096)
    h.timing_enable(64)
    mw = 3
    while True:
        g = partition_grammar(rng, 8, n_cmd=4)
        if accepts(g, [0, 1]):                          # slot 1 is command 0, slot 6 command 1
            break
    N16 = np.full(B, 2, np.uint32)
    for S, g, n in ((8, g, N), (16, partition_grammar(rng, 16, n_cmd=4), N16)):
        cuts = record_cuts(n, S)
        print("S %d: %d sequences, record launches at %s, %d kernel launches" % (S, B, cuts, gram_launches(cuts)))
        assert cuts == ([0, B] if S == 8 else [0, SEQ_CHUNK, B]) and gram_launches(cuts) == 2
        f = feat if S == 8 else _poisoned(rng, n, 2)
        w0 = _prefill_words(B, mw)
        got = h.connected_grammar(f, n, g, 0, mw, words=w0.copy())
        assert _count(h, TAG_GRAM) == 2
        ww, wn, wt = go.decode(f, n, bank, 13, 4096, g, 0, mw, nthreads=NTHREADS)
        assert np.array_equal(got[1], wn) and np.array_equal(got[2], wt), S
        _check_words(got[0], ww, wn, w0)
        if S == 8:
            _check_plants(got, plant, mw)
        for lo, hi in ((0, SEQ_CHUNK), (SEQ_CHUNK, B)):
            part = h.connected_grammar(f[lo:hi], n[lo:hi], g, 0, mw, words=w0[lo:hi].copy())
            assert _count(h, TAG_GRAM) == 1
            for a, b in zip(part, got):
                _equal_rows(a, b[lo:hi], "S %d slice %d..%d" % (S, lo, hi))
    h.close()
