"""Live streams of any length (include/sr_long_stream.h, K14 in csrc/sr_long_stream.cu): the long-form VAD carried across
pushes, one decision per segment as it closes.

The definition is prefix equality: after any push, a stream's events so far are the closed records of
sr_recognise_long_batch on the n samples pushed to it, its open segment is that call's trailing open record and its atap
is the call's atap. sr_recognise_long_batch is pinned to the oracle by test_long.py, so every GPU test here compares
against it, bit for bit, on the same prefix.

CPU: a header guard; the ring bound by brute force (every sample get_mfcc reads, x[-1] included, is in the ring and in the
row when a segment is recognised, for both geometries, every decodable length, every closing position relative to a
push boundary and several chunk lengths); long_fsm_window's carried state over windows of any length, cut anywhere.
GPU: chunk lengths 1 ... max_chunk and random ragged pushes (0 and a late start included), planted push / window / ring
edges, 119- and 120-frame segments in both geometries, segments on and across the ring's wrap, an open segment longer
than the ring, calibration lengths, the digit recordings in 10 ms and 80 ms chunks, one stream of 2^27 samples beside 4 095
short ones, subset resets, the matcher / bank / geometry switched between pushes, the 2^32 - 1 sample limit, composition
with sr_streams_*, the caller's event buffer, the launch count and threads."""
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = ("digits_1_10_a", "digits_1_10_b", "digits_1_9_units_a", "digits_1_9_units_b")
NULL = 0xFFFFFFFF
ST_OK, ST_VAD_FAIL, ST_MFCC_FAIL = 0, 1, 2
HEADER = open(os.path.join(ROOT, "include", "sr_long_stream.h")).read()
HISTORY, MIRROR = (int(re.search(r"#define SR_LONG_STREAM_%s\s+(\d+)u" % k, HEADER).group(1)) for k in ("HISTORY", "MIRROR"))
FRAME_LEN = {0: 160, 1: 200}                # frame length per geometry
REC = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


# ---- the pool's sizes, restated from the header (the GPU tests check ring_len against the pool's own R) --------------------
def ring_len(max_chunk, n_len):
    return -(-(max(n_len, HISTORY) + max_chunk) // 80) * 80


def window(max_chunk):
    return min(1024, -(-max_chunk // 80))


def events_per_push(max_chunk, n_len):
    c = n_len if n_len and n_len % 240 == 0 else 0
    return -(-(-(-(max_chunk + c) // 80)) // 19)


def frames_of(n):
    return -(-(n - 160) // 80) if n > 160 else 0


def decodable(length, geom):
    fl = FRAME_LEN[geom]
    return length >= fl and (length - fl) // 80 + 1 <= 119


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_every_long_stream_entry_point_is_run_here():
    """every entry point of include/sr_long_stream.h is called by a GPU test of this file"""
    hdr = open(os.path.join(ROOT, "include", "sr_long_stream.h")).read()
    names = set(re.findall(r"\b(?:int|uint32_t)\s+(sr_\w+)\s*\(", hdr))
    py = {"sr_long_streams_create": "LongStreamPool(", "sr_long_streams_destroy": ".close()",
          "sr_long_streams_reset": ".reset(", "sr_long_streams_push": ".push(", "sr_long_streams_push_ragged": ".push_ragged(",
          "sr_long_streams_fetch": ".fetch(", "sr_long_streams_pending": ".pending()",
          "sr_long_streams_max_events": ".max_events", "sr_long_streams_ring_len": ".ring_len",
          "sr_long_streams_state": ".state()"}
    assert names == set(py), names
    src = open(os.path.abspath(__file__)).read()
    gpu = src[src.index("# ---- GPU"):]
    for n in names:
        assert gpu.count(py[n]) >= 1, n


def _mapped_start(st, R):
    ms = st % R
    return R if ms == 0 and st != 0 else ms


@pytest.mark.parametrize("geom", [0, 1])
def test_ring_holds_every_sample_a_decodable_segment_reads(geom):
    assert (HISTORY, MIRROR) == (10561, 9680)            # the derivation below: 9 680 + 881, and the longest segment
    fl = FRAME_LEN[geom]
    lengths = [L for L in range(720, 12000, 80) if decodable(L, geom)]
    assert max(lengths) == (9600 if geom == 0 else 9680) and not decodable(max(lengths) + 80, geom)
    for max_chunk in (1, 79, 80, 81, 777, 4096, 1 << 20):
        for n_len in (0, 2400, 65520):
            R = ring_len(max_chunk, n_len)
            assert R % 80 == 0 and R >= max_chunk + HISTORY and R >= n_len + max_chunk
            for c in sorted(v for v in {1, 79, 80, 81, 777, max_chunk // 2 + 1, max_chunk} if v <= max_chunk):
                d = np.arange(min(c, 4096), dtype=np.int64)
                if c > 4096:
                    d = np.concatenate([d, np.arange(c - 4096, c, dtype=np.int64)])
                for L in lengths:
                    F = (L - fl) // 80 + 1
                    end = 10 ** 6 * 80 + 80                         # any end; the ring holds [n - R, n) after the push
                    st = end - L
                    n_prev = end + 880 - d                          # the segment is not reported before this push ...
                    n = n_prev + c                                  # ... and is by it (n >= end + 881)
                    assert (n >= end + 881).all()
                    first, last = st - 1, st + 80 * (F - 1) + fl    # get_mfcc reads [start - 1, last)
                    assert (first >= n - R).all() and last <= end
    # the row: every read of a decodable segment lies in [0, R + M), slot by slot, for every start in a ring period
    for max_chunk, n_len in ((1, 0), (640, 2400), (777, 65520)):
        R = ring_len(max_chunk, n_len)
        for L in lengths:
            F = (L - fl) // 80 + 1
            for st in [j * R + 80 * d for j in (1, 2) for d in range(-125, 3)]:
                ms = _mapped_start(st, R)
                pos = ms + np.arange(-1, 80 * (F - 1) + fl)
                off = st + np.arange(-1, 80 * (F - 1) + fl)
                assert pos[0] >= 0 and pos[-1] < R + MIRROR and ms + L <= R + MIRROR
                assert ((pos % R) == (off % R)).all()           # ring slot, or its mirror behind the ring
                assert (pos[pos >= R] - R < MIRROR).all()
            assert _mapped_start(0, R) == 0                     # stream sample 0: x[-1] pinned to mid_val, as the batch


def fsm_seq(act):
    """the sequential FSM of VAD.C:164-216: [(start, end)], end NULL while open"""
    cur = front = back = 0
    segs = []
    for k, a in enumerate(act):
        if a:
            if cur == 0:
                cur, front = 1, 1
            elif cur == 1:
                front += 1
                if front >= 8:
                    cur, front = 2, 0
                    segs.append([80 * (k - 7), NULL])
            elif cur == 3:
                back, cur = 0, 2
        else:
            if cur == 2:
                cur, back = 3, 1
            elif cur == 3:
                back += 1
                if back >= 11:
                    cur, back = 0, 0
                    segs[-1][1] = 80 * (k - 11) + 160
            elif cur == 1:
                front, cur = 0, 0
    return [tuple(s) for s in segs]


def fsm_cut(act, cuts):
    """long_fsm_window restated, over windows cut at `cuts` (any lengths >= 1)"""
    op, run, segs = False, 0, []

    def event(frame):
        if op:
            segs[-1][1] = 80 * frame + 80
        else:
            segs.append([80 * frame, NULL])
    bounds = [0] + sorted(cuts) + [len(act)]
    for base, top in zip(bounds, bounds[1:]):
        a = list(act[base:top])
        nw, cur, ev = len(a), 0, False
        if nw == 0:
            continue
        if run:
            need, want = (11 if op else 8) - run, 0 if op else 1
            if need <= nw and a[:need] == [want] * need:
                event(base - run)
                op, cur, ev = not op, need, True
        while True:
            L, want = (11, 0) if op else (8, 1)
            p = next((p for p in range(cur, nw - L + 1) if a[p:p + L] == [want] * L), -1)
            if p < 0:
                break
            event(base + p)
            op, cur, ev = not op, p + L, True
        brk = 1 if op else 0
        last_brk = max((i for i in range(nw) if a[i] == brk), default=-1)
        if not ev and last_brk < 0:
            run += nw
        else:
            f = max(last_brk + 1, cur)
            run = nw - f if f < nw else 0
    return [tuple(s) for s in segs]


def test_fsm_carried_over_windows_of_any_length():
    """push windows are as short as one frame: the carried run may span many windows before it completes or breaks"""
    rng = np.random.default_rng(14)
    for trial in range(3000):
        n = int(rng.integers(1, 90))
        runs = rng.integers(1, 15, 40)
        act = np.repeat(np.arange(40) % 2 == trial % 2, runs)[:n].astype(int).tolist()
        k = int(rng.integers(0, n))
        cuts = set(rng.choice(np.arange(1, n), size=min(k, n - 1), replace=False).tolist()) if n > 1 else set()
        assert fsm_cut(act, cuts) == fsm_seq(act), (act, cuts)
        assert fsm_cut(act, set(range(1, n))) == fsm_seq(act)


# ---- planted inputs ------------------------------------------------------------------------------------------------------
def planted_atap(S=1):
    """under this atap every sample is below b_thl (mid - n_thl wraps), so no band crossing counts; a loud block (2 148)
    sums |x - mid| = 8 000 and a frame is active exactly when both its blocks are loud (as planted() in test_long.py)"""
    a = np.zeros(S, sr_b200.ATAP_DTYPE)
    a["mid_val"], a["n_thl"], a["z_thl"], a["s_thl"] = 2048, 5000, 2, 15999
    return a


QUIET, LOUD, MARK = 2000, 2148, 4095


def plant_segs(n_blocks, segs):
    """n_blocks quiet blocks with loud blocks p .. p + a for each (p, a): a segment [80p, 80(p + a) + 80) of a active
    frames, closed by the quiet blocks after it. Under planted_atap a frame sums 7 680 over two quiet blocks, 11 840 over a
    quiet and a loud one and 16 000 over two loud ones (s_thl 15 999). Quiet samples differ from mid_val (2 048), and the
    sample before each segment (its x[-1], in a quiet block) is MARK: get_mfcc's pre-emphasis of the segment's first sample
    then tells the real x[-1] from the mid_val that is pinned at row offset 0. A marked quiet block sums 5 839, so a frame
    over it stays inactive."""
    x = np.full(80 * n_blocks, QUIET, np.uint16)
    for p, a in segs:
        x[80 * p:80 * (p + a + 1)] = LOUD
        if p:
            x[80 * p - 1] = MARK
    return x


def plant_act(act):
    """PCM whose frames are active exactly where act is 1 (blocks k, k + 1 loud <=> frame k active), under planted_atap;
    an isolated active frame is two loud blocks, so act is first widened into the frames it forces"""
    act = np.asarray(act, bool)
    loud = np.zeros(len(act) + 1, bool)
    loud[:-1] |= act
    loud[1:] |= act
    return np.repeat(np.where(loud, LOUD, QUIET).astype(np.uint16), 80)


# ---- the prefix definition -----------------------------------------------------------------------------------------------
def expected(h, xs, ns, n_len, atap0, rows=None):
    """sr_recognise_long_batch on the prefix xs[s][:ns[s]] of each stream: per stream (closed records, open start, atap)"""
    rows = range(len(xs)) if rows is None else rows
    rows = [s for s in rows]
    U = max(1, max(int(ns[s]) for s in rows))
    pcm = np.zeros((len(rows), U), np.uint16)
    lens = np.zeros(len(rows), np.uint32)
    for i, s in enumerate(rows):
        pcm[i, :ns[s]] = xs[s][:ns[s]]
        lens[i] = ns[s]
    atap = np.zeros(len(rows), sr_b200.ATAP_DTYPE) if atap0 is None else np.ascontiguousarray(atap0[rows])
    max_segs = int(lens.max()) // (19 * 80) + 4              # closings are >= 19 frames apart
    r = h.recognise_long_batch(pcm, max_segs, n_len, lens, atap)
    out = {}
    for i, s in enumerate(rows):
        k = int(r["n_segs"][i])
        assert k <= max_segs
        recs = [tuple(int(v) for v in rec) for rec in r["segs"][i, :k].tolist()]
        closed = [t for t in recs if t[2] != ST_VAD_FAIL]
        op = recs[-1][0] if recs and recs[-1][2] == ST_VAD_FAIL else NULL
        out[s] = (closed, op, r["atap"][i].tobytes())
    return out


class Feed:
    """a pool and its streams: pushes, collects each stream's events in order, checks prefix equality"""

    def __init__(self, h, xs, max_chunk, n_len=0, atap0=None):
        self.h, self.xs, self.n_len = h, [np.asarray(x, np.uint16) for x in xs], n_len
        self.S = len(xs)
        self.atap0 = atap0
        self.pool = sr_b200.LongStreamPool(h, self.S, max_chunk, n_len, atap0)
        self.n = np.zeros(self.S, np.int64)
        self.got = [[] for _ in range(self.S)]

    def take(self, evs):
        for e in evs:
            assert e["segment"] == len(self.got[e["stream"]]), e
            self.got[e["stream"]].append(tuple(int(e[k]) for k in REC))

    def push(self, lens):
        lens = np.asarray(lens, np.int64)
        width = max(1, int(lens.max()))
        chunk = np.zeros((self.S, width), np.uint16)
        for s in range(self.S):
            seg = self.xs[s][self.n[s]:self.n[s] + lens[s]]
            assert len(seg) == lens[s]
            chunk[s, :lens[s]] = seg
        self.take(self.pool.push_ragged(chunk, lens.astype(np.uint32)))
        self.n += lens

    def check(self, rows=None):
        st = self.pool.state()
        assert (st["n_recv"] == self.n).all()
        rows = [s for s in (range(self.S) if rows is None else rows)
                if self.n[s] > 0 and (self.n[s] >= self.n_len or not (self.n_len and self.n_len % 240 == 0))]
        if not rows:
            return
        want = expected(self.h, self.xs, self.n, self.n_len, self.atap0, rows)
        for s in rows:
            closed, op, atap = want[s]
            assert self.got[s] == closed, (s, int(self.n[s]), self.got[s][-3:], closed[-3:])
            assert int(st["n_closed"][s]) == len(closed)
            assert int(st["open_start"][s]) == op, (s, int(self.n[s]))
            assert st["atap"][s].tobytes() == atap, s

    def close(self):
        self.pool.close()


def _drive(feed, schedule, every=1):
    for i, lens in enumerate(schedule):
        feed.push(lens)
        if every and (i % every == 0 or i == len(schedule) - 1):
            feed.check()


def _uniform(total, c):
    out, n = [], 0
    while n < total:
        out.append(min(c, total - n))
        n += out[-1]
    return out


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bank():
    return ox.synth_bank()


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 79, 80, 81, 159, 160, 161, 777, 1000])
def test_chunk_lengths(handle, bank, c):
    handle.set_bank(bank[0], bank[1], 4096)
    max_chunk = 1000
    if c == 1:      # planted, short: a segment at sample 0, a closing at every phase of nothing but single samples
        xs = [plant_segs(60, [(0, 9)]), plant_segs(70, [(3, 12), (35, 8)])]
        f = Feed(handle, xs, max_chunk, 0, planted_atap(2))
        _drive(f, [[1, 1]] * len(xs[0]) + [[0, 1]] * (len(xs[1]) - len(xs[0])), every=7)
    else:
        xs = list(ox.synth_long(3, 24000, 0x14C0 + c))
        f = Feed(handle, xs, max_chunk, 2400)
        _drive(f, [[k] * 3 for k in _uniform(24000, c)], every=1 if c >= 79 else 0)
    f.check()
    assert sum(len(g) for g in f.got) > 0
    f.close()


@pytest.mark.gpu
def test_random_ragged_pushes(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(141)
    S, N, max_chunk = 8, 40000, 700
    xs = list(ox.synth_long(S, N, 0x14D0))
    f = Feed(handle, xs, max_chunk, 2400)
    start = np.zeros(S, int)
    start[3] = 20                                       # a stream that starts late
    i = 0
    while (f.n < N).any():
        lens = rng.integers(0, max_chunk + 1, S)
        lens[rng.random(S) < 0.2] = 0
        lens[i < start] = 0
        lens = np.minimum(lens, N - f.n)
        f.push(lens)
        f.check()
        i += 1
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("max_chunk", [80, 777])
def test_planted_activity_across_push_and_window_edges(handle, bank, max_chunk):
    """runs of 6-13 frames (both sides of 8 and 11) cut by pushes and by windows of W frames at once"""
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(max_chunk)
    S = 6
    xs = []
    for s in range(S):
        runs = rng.integers(6, 14, 120)
        act = np.repeat(np.arange(120) % 2 == s % 2, runs).astype(int)
        xs.append(plant_act(act))
    f = Feed(handle, xs, max_chunk, 0, planted_atap(S))
    W = window(max_chunk)
    N = min(len(x) for x in xs)
    while (f.n < N).any():
        lens = np.array([int(rng.choice([1, 80 * W - 1, 80 * W, 80 * W + 1, max_chunk, int(rng.integers(0, max_chunk + 1))]))
                         for _ in range(S)])
        lens = np.minimum(np.minimum(lens, max_chunk), N - f.n)
        f.push(lens)
        f.check()
    assert sum(len(g) for g in f.got) > 100
    f.close()


@pytest.mark.gpu
def test_closing_at_end_plus_880_and_881(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    x = plant_segs(80, [(5, 20)])
    end = 80 * 25 + 80
    for first in (end + 880, end + 881):
        f = Feed(handle, [x], 4000, 0, planted_atap())
        f.push([first])
        f.check()
        assert len(f.got[0]) == (1 if first == end + 881 else 0)
        f.push([1])
        f.check()
        assert len(f.got[0]) == 1 and f.got[0][0][:2] == (80 * 5, end)
        f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [0, 1])
def test_frame_caps_and_ring_wrap(handle, bank, geom):
    """119- and 120-frame segments; decodable segments starting on ring slot 0 (x[-1] in slot R - 1), on the ring's last
    block and across the wrap; one open longer than the ring that closes much later; one at stream sample 0.
    Segment starts are multiples of 80 and so is R, so no start lies on slot R - 1: the ring's last block (slot R - 80)
    stands in for it. Every segment's x[-1] is MARK, so reading mid_val instead of slot R - 1 changes the features."""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_geometry(geom)
    try:
        max_chunk = 640
        probe = sr_b200.LongStreamPool(handle, 1, max_chunk, 0)
        assert probe.ring_len == ring_len(max_chunk, 0)
        probe.close()
        R = ring_len(max_chunk, 0) // 80                            # in blocks
        a119 = 119 if geom == 0 else 120                           # active frames of a 119-frame segment: len 80 (a + 1)
        segs = [(0, 30), (R, 40), (2 * R - 1, 40), (3 * R - 20, 60),    # sample 0; slot 0; last block; across the wrap
                (4 * R, a119), (4 * R + 150, a119 + 1),                  # 119 frames; 120 frames
                (6 * R + 7, 3 * R)]                                      # longer than the ring
        x = plant_segs(11 * R, segs)
        rng = np.random.default_rng(geom)
        f = Feed(handle, [x, x[:len(x) // 2].copy()], max_chunk, 0, planted_atap(2))
        while f.n[0] < len(x):
            c = int(rng.integers(1, max_chunk + 1))
            f.push([min(c, len(x) - f.n[0]), min(c, len(x) // 2 - f.n[1])])
            if rng.random() < 0.1:
                f.check()
        f.check()
        got = f.got[0]
        assert [g[:2] for g in got] == [(80 * p, 80 * (p + a) + 80) for p, a in segs]
        frm = [g[3] for g in got]
        assert frm[4] == 119 and frm[5] == 0 and got[5][2] == ST_MFCC_FAIL and frm[6] == 0 and got[6][2] == ST_MFCC_FAIL
        assert all(g[2] == ST_OK for i, g in enumerate(got) if i not in (5, 6))
        R80 = 80 * R
        assert got[1][0] % R80 == 0 and got[2][0] % R80 == R80 - 80 and got[3][0] % R80 + 80 * 61 > R80   # where they sit
    finally:
        handle.set_geometry(0)
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_len", [2400, 0, 2401, 65520])
@pytest.mark.parametrize("given", [True, False])
def test_calibration_lengths(handle, bank, n_len, given):
    handle.set_bank(bank[0], bank[1], 4096)
    S, N, max_chunk = 3, 90000, 500
    xs = list(ox.synth_long(S, N, 0x14E0 + n_len))
    atap0 = None
    if given:
        atap0 = np.zeros(S, sr_b200.ATAP_DTYPE)
        atap0["mid_val"], atap0["n_thl"], atap0["z_thl"], atap0["s_thl"] = 2040, 60, 2, 9000
    f = Feed(handle, xs, max_chunk, n_len, atap0)
    assert f.pool.ring_len == ring_len(max_chunk, n_len)
    rng = np.random.default_rng(n_len)
    i = 0
    while (f.n < N).any():
        f.push(np.minimum(rng.integers(0, max_chunk + 1, S), N - f.n))
        if i % 9 == 0:
            f.check()
        i += 1
    f.check()
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("c", [80, 640])
def test_digit_recordings(handle, bank, c):
    handle.set_bank(bank[0], bank[1], 4096)
    xs = [ox.golden_wav(n) for n in FIXTURES]
    f = Feed(handle, xs, 640, 2400)
    N = np.array([len(x) for x in xs])
    while (f.n < N).any():
        f.push(np.minimum(c, N - f.n))
    f.check()
    assert [len(g) for g in f.got] == [10, 10, 13, 13]
    f.close()


@pytest.mark.gpu
def test_one_stream_of_2_27_samples_beside_4095_short_ones(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    S, max_chunk, short = 4096, 1 << 16, 20000
    big = ox.synth_long(1, 1 << 27, 0x14F0)[0]
    small = ox.synth_long(S - 1, short, 0x14F1)
    pool = sr_b200.LongStreamPool(handle, S, max_chunk, 2400)
    got = [[] for _ in range(S)]
    chunk = sr_b200.host_alloc_dev(0, S * max_chunk * 2)
    buf, ptr = chunk[0].view(np.uint16).reshape(S, max_chunk), chunk[1]
    try:
        n = 0
        rng = np.random.default_rng(5)
        sn = np.zeros(S, np.int64)
        while n < (1 << 27):
            lens = np.zeros(S, np.uint32)
            lens[0] = min(max_chunk, (1 << 27) - n)
            buf[0, :lens[0]] = big[n:n + lens[0]]
            ls = np.minimum(rng.integers(0, 3000, S - 1), short - sn[1:]).astype(np.uint32)
            for s in np.flatnonzero(ls):
                buf[s + 1, :ls[s]] = small[s, sn[s + 1]:sn[s + 1] + ls[s]]
            lens[1:] = ls
            for e in pool.push_ragged(ptr, lens, stride=max_chunk):
                assert e["segment"] == len(got[e["stream"]])
                got[e["stream"]].append(tuple(int(e[k]) for k in REC))
            sn += lens
            n += int(lens[0])
        assert (sn[1:] == short).all()
        st = pool.state()
        assert int(st["n_recv"][0]) == 1 << 27
        want = expected(handle, [big], [1 << 27], 2400, None)[0]
        assert got[0] == want[0] and len(got[0]) > 1000
        assert int(st["open_start"][0]) == want[1] and st["atap"][0].tobytes() == want[2]
        ws = expected(handle, list(small), [short] * (S - 1), 2400, None)
        for s in range(S - 1):
            assert got[s + 1] == ws[s][0], s
    finally:
        pool.close()
        sr_b200.host_free(ptr)


@pytest.mark.gpu
def test_reset_a_subset_mid_stream(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    S, N, c = 6, 50000, 640
    xs = list(ox.synth_long(S, N, 0x1500))
    atap_r = np.zeros(S, sr_b200.ATAP_DTYPE)
    atap_r["mid_val"] = 77
    f = Feed(handle, xs, c, 2400)
    for k in _uniform(N // 2 + 123, c):
        f.push([k] * S)
    which = np.zeros(S, np.uint8)
    which[[1, 4]] = 1
    f.pool.reset(which, atap_r)
    cut = int(f.n[1])
    for s in (1, 4):                                    # the reset streams now restart from sample `cut`
        f.xs[s] = f.xs[s][cut:].copy()
        f.n[s] = 0
        f.got[s] = []
    f.atap0 = atap_r.copy()
    f.atap0[[0, 2, 3, 5]] = 0
    while (f.n[[0, 2, 3, 5]] < N).any():
        lens = np.minimum(c, np.array([len(x) for x in f.xs]) - f.n)
        f.push(lens)
    f.check()
    f.close()


@pytest.mark.gpu
def test_matcher_bank_and_geometry_switched_between_pushes(handle, bank):
    bank2 = ox.synth_bank(9, 0x7E3B0000)
    S, N, c = 4, 60000, 800
    xs = list(ox.synth_long(S, N, 0x1510))
    configs = [(0, 0, 0, bank), (1, 0, 0, bank2), (0, 2, 8, bank), (0, 0, 0, None), (1, 2, 118, bank2)]
    f = Feed(handle, xs, c, 2400)
    rng = np.random.default_rng(7)
    try:
        for i, k in enumerate(_uniform(N, c)):
            geom, flags, r, b = configs[int(rng.integers(len(configs)))]
            handle.set_geometry(geom)
            handle.set_match(flags, r)
            if b is None:
                handle.set_bank(np.zeros((0, 4096), np.uint8), 0, 4096)
            else:
                handle.set_bank(b[0], b[1], 4096)
            before = [len(g) for g in f.got]
            f.push([k] * S)
            if any(len(g) > n0 for g, n0 in zip(f.got, before)):
                want = expected(handle, f.xs, f.n, 2400, None)      # under this push's settings
                for s in range(S):
                    assert f.got[s][before[s]:] == want[s][0][before[s]:len(f.got[s])], (i, s)
        assert sum(len(g) for g in f.got) > 10
    finally:
        handle.set_geometry(0)
        handle.set_match(0, 0)
    f.close()


@pytest.mark.gpu
def test_stream_of_2_32_minus_1_samples(handle, bank):
    """a stream taken to 2^32 - 1 samples (quiet, then a planted segment near the end); the push that would pass the
    limit fails and changes nothing"""
    handle.set_bank(bank[0], bank[1], 4096)
    max_chunk = 1 << 20
    pool = sr_b200.LongStreamPool(handle, 1, max_chunk, 0, planted_atap())
    lim = (1 << 32) - 1
    tail_len = 80 * 4000
    tail = plant_segs(4000, [(100, 30), (1000, 50), (2500, 9)])
    base = (lim - tail_len) // 80 * 80                  # the tail starts on a block, after quiet samples only
    quiet = np.full((1, max_chunk), QUIET, np.uint16)
    got = []
    try:
        n = 0
        while n < base:
            k = min(max_chunk, base - n)
            got += pool.push(quiet[:, :k])
            n += k
        assert got == []
        rest = np.concatenate([tail, np.full(lim - base - tail_len, QUIET, np.uint16)])
        for i in range(0, len(rest), max_chunk):
            got += pool.push(np.ascontiguousarray(rest[None, i:i + max_chunk]))
        st = pool.state()
        assert int(st["n_recv"][0]) == lim
        want = expected(handle, [rest], [len(rest)], 0, planted_atap())[0][0]
        assert [(e["start"] - base, e["end"] - base) + tuple(e[k] for k in REC[2:]) for e in got] == want
        assert len(want) == 3
        with pytest.raises(sr_b200.SrError):
            pool.push(np.full((1, 1), 2148, np.uint16))
        with pytest.raises(sr_b200.SrError):
            pool.push_ragged(np.full((1, 2), 2148, np.uint16), [2])
        st2 = pool.state()
        for k in st:
            assert st2[k].tobytes() == st[k].tobytes(), k
        assert pool.push(np.zeros((1, 1), np.uint16)[:, :0]) == []
        with pytest.raises(sr_b200.SrError):                # lens[s] > max_chunk fails before any stream changes
            pool.push_ragged(np.zeros((1, max_chunk + 1), np.uint16), [max_chunk + 1])
    finally:
        pool.close()


@pytest.mark.gpu
def test_composition_with_fixed_capture_streams(handle, bank):
    """on streams of <= 65 535 samples, after the last push, segments 0-2 equal sr_streams_* events field for field"""
    handle.set_bank(bank[0], bank[1], 4096)
    S, N, c = 16, 65535, 800
    xs = ox.synth_long(S, N, 0x1520)
    k4 = sr_b200.StreamPool(handle, S, N, 2400)
    f = Feed(handle, list(xs), c, 2400)
    old = []
    n = 0
    while n < N:
        k = min(c, N - n)
        old += k4.push(np.ascontiguousarray(xs[:, n:n + k]))
        f.push([k] * S)
        n += k
    k4.close()
    for s in range(S):
        mine = [dict(zip(REC, g), stream=s, segment=i) for i, g in enumerate(f.got[s][:3])]
        theirs = sorted([e for e in old if e["stream"] == s], key=lambda e: e["segment"])
        assert mine == theirs, s
    f.check()
    f.close()


@pytest.mark.gpu
def test_event_buffer_footprint_and_queue(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    S, N, c = 8, 40000, 640
    xs = ox.synth_long(S, N, 0x1530)
    ref = sr_b200.LongStreamPool(handle, S, c, 2400)
    pool = sr_b200.LongStreamPool(handle, S, c, 2400)
    assert pool.max_events == S * events_per_push(c, 2400)
    all_ref, all_got, queued = [], [], 0
    buf = (sr_b200.StreamEvent * 64)()
    try:
        for i, k in enumerate(_uniform(N, c)):
            chunk = np.ascontiguousarray(xs[:, i * c:i * c + k])
            all_ref += ref.push(chunk)
            C.memset(buf, 0x5A, C.sizeof(buf))
            m = 1 if i % 3 else 0
            ne = pool.push(chunk, max_events=m, events=buf)
            raw = bytes(buf)
            rec = C.sizeof(sr_b200.StreamEvent)
            assert ne <= m
            assert raw[ne * rec:] == b"\x5A" * (len(raw) - ne * rec)      # nothing past the n_events records
            all_got += pool._events(ne, buf)
            queued = max(queued, pool.pending())
        assert queued > 0
        all_got += pool.fetch()
        assert pool.pending() == 0
        # events of one push come in no fixed order across streams; each stream's come oldest first
        assert len(all_got) == len(all_ref) > 10
        for s in range(S):
            assert [e for e in all_got if e["stream"] == s] == [e for e in all_ref if e["stream"] == s], s
    finally:
        ref.close()
        pool.close()


@pytest.mark.gpu
def test_launches_per_push_are_fixed(handle, bank):
    S, c = 32, 640
    xs = ox.synth_long(S, 32000, 0x1540)
    pool = sr_b200.LongStreamPool(handle, S, c, 2400)
    try:
        for with_bank in (True, False):
            if with_bank:
                handle.set_bank(bank[0], bank[1], 4096)
            else:
                handle.set_bank(np.zeros((0, 4096), np.uint8), 0, 4096)
            pool.reset()
            for i in range(0, 32000, c):
                before = handle.launch_count()
                pool.push(np.ascontiguousarray(xs[:, i:i + c]))
                assert handle.launch_count() - before == (5 if with_bank else 4)
    finally:
        pool.close()


@pytest.mark.gpu
def test_threads_beside_a_long_batch_handle(bank):
    S, N, c = 8, 30000, 640
    xs = ox.synth_long(S, N, 0x1550)
    rec = ox.synth_long(4, 200000, 0x1551)

    def job_pool(h):
        h.set_bank(bank[0], bank[1], 4096)
        p = sr_b200.LongStreamPool(h, S, c, 2400)
        evs = []
        for i in range(0, N, c):
            evs += p.push(np.ascontiguousarray(xs[:, i:i + c]))
        p.close()
        return sorted(evs, key=lambda e: (e["stream"], e["segment"]))   # no fixed order across streams within a push

    def job_batch(h):
        h.set_bank(bank[0], bank[1], 4096)
        r = h.recognise_long_batch(rec, 512, 2400)
        return r["segs"].tobytes() + r["n_segs"].tobytes()

    jobs = [job_pool, job_pool, job_batch]
    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        serial = [j(h) for j, h in zip(jobs, handles)]
        for rep in range(3):
            out = [None] * len(jobs)

            def run(i):
                out[i] = jobs[i](handles[i])
            th = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert out == serial, rep
    finally:
        for h in handles:
            h.close()


# ---- the event buffer at its bound ---------------------------------------------------------------------------------------
# Period-19 activity: 8 active frames, then 11 inactive. A run of 8 opens a segment on its 8th frame and the 11th inactive
# frame after it closes the segment, so closings fall every 19 frames, the densest the FSM allows, and a push that
# evaluates F new frames starting on a closing closes exactly ceil(F / 19) segments per stream: the header's E.
def period_act(n_frames, offset):
    """offset inactive frames, then runs of 8 active and 11 inactive frames"""
    k = np.arange(n_frames) - offset
    return ((k >= 0) & (k % 19 < 8)).astype(np.uint8)


def period_closings(n_frames, offset):
    """the frames on which period_act's segments close: the 11th inactive frame after each run"""
    return np.arange(offset + 18, n_frames, 19)


def closings_between(closings, n0, n1):
    """segments a push from n0 to n1 samples closes: closing frames it evaluates, frames_of(n0) .. frames_of(n1) - 1"""
    return int(((closings >= frames_of(n0)) & (closings < frames_of(n1))).sum())


def test_period_19_string_closes_every_19_frames():
    """the sequential FSM on period_act closes on period_closings for every offset, and the planted PCM realises the
    string under planted_atap (the long-form VAD oracle on the PCM gives the FSM's segments)"""
    lo = ox.long_oracle()
    for j in range(19):
        act = period_act(600, j)
        x = plant_act(act)
        segs = fsm_seq(act[:frames_of(len(x))])                     # the frames the PCM's length evaluates
        closed = [s for s in segs if s[1] != NULL]
        assert [(e - 160) // 80 + 11 for _, e in closed] == period_closings(frames_of(len(x)), j).tolist()
        n, seg = lo.vad_long(x[None, :], planted_atap(), 64)
        assert [tuple(s) for s in seg[0, :int(n[0])].tolist()] == segs, j
    assert events_per_push(1 << 20, 0) == 690 and (-(-(1 << 20) // 80)) // 19 == 689    # ceil and floor differ here


def _take_counts(f, lens, max_events=None):
    """one ragged push of Feed f: (events handed out, per-stream events handed out)"""
    before = [len(g) for g in f.got]
    lens = np.asarray(lens, np.int64)
    chunk = np.zeros((f.S, max(1, int(lens.max()))), np.uint16)
    for s in range(f.S):
        chunk[s, :lens[s]] = f.xs[s][f.n[s]:f.n[s] + lens[s]]
    evs = f.pool.push_ragged(chunk, lens.astype(np.uint32), max_events=max_events)
    f.take(evs)
    f.n += lens
    return len(evs), [len(g) - b for g, b in zip(f.got, before)]


def _check_prefix(f):
    """with events still queued, each stream's events so far are a prefix of the closed records, and n_closed counts
    them all"""
    st = f.pool.state()
    want = expected(f.h, f.xs, f.n, f.n_len, f.atap0)
    for s in range(f.S):
        closed = want[s][0]
        assert f.got[s] == closed[:len(f.got[s])], s
        assert int(st["n_closed"][s]) == len(closed) and int(st["n_recv"][s]) == f.n[s]


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [0, 1])
def test_event_buffer_at_its_bound_without_calibration(handle, bank, geom):
    """max_chunk = 2^20, n_len = 0: 19 streams of period-19 activity offset by 0 ... 18 frames (every phase of the carried
    run meets every push and window edge), pushes of 2^20 samples and ragged shorter ones; each stream closes exactly the
    segments its phase puts into each push, and prefix equality holds after every push"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_geometry(geom)
    max_chunk, S = 1 << 20, 19
    sched = [max_chunk, 80 * 4099 + 41, max_chunk, max_chunk - 1, 12345, max_chunk]
    total = sum(sched) + 80 * 19
    n_frames = total // 80 + 2
    xs = [plant_act(period_act(n_frames, j)) for j in range(S)]
    clos = [period_closings(n_frames, j) for j in range(S)]
    f = Feed(handle, xs, max_chunk, 0, planted_atap(S))
    try:
        E = events_per_push(max_chunk, 0)
        assert f.pool.max_events == S * E == S * 690
        rng = np.random.default_rng(geom)
        for i, c in enumerate(sched):
            lens = np.full(S, c, np.int64)
            if i == 4:                                              # ragged: a different edge for every stream
                lens = rng.integers(0, c + 1, S)
            want = [closings_between(clos[s], f.n[s], f.n[s] + lens[s]) for s in range(S)]
            n, per = _take_counts(f, lens)
            assert per == want and n == sum(want), (i, per, want)
            f.check()
        assert max(closings_between(clos[s], 0, f.n[s]) for s in range(S)) > 2000
    finally:
        handle.set_geometry(0)
        f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("small_buffer", [False, True])
def test_event_buffer_filled_to_cap(handle, bank, small_buffer):
    """every stream aligned: the first push ends just before a closing frame, so the next push of 2^20 samples evaluates
    13 108 frames from a closing on and closes E = 690 segments per stream: it hands out exactly max_events events (the
    device buffer full to cap). With a caller buffer of 1 000 events, more than cap events carry over to the next push and
    to fetch, oldest first"""
    handle.set_bank(bank[0], bank[1], 4096)
    max_chunk, S = 1 << 20, 19
    first = 80 * (19 * 10 + 18) + 160                               # frames_of(first) = 208: frame 208 closes
    assert frames_of(first) == 208 and 208 in period_closings(300, 0)
    n_frames = (first + 3 * max_chunk) // 80 + 2
    x = plant_act(period_act(n_frames, 0))
    f = Feed(handle, [x] * S, max_chunk, 0, planted_atap(S))
    clos = period_closings(n_frames, 0)
    try:
        cap = f.pool.max_events
        assert cap == S * 690
        m = 1000 if small_buffer else None
        produced = handed = 0
        for i, c in enumerate((first, max_chunk, max_chunk)):
            k = closings_between(clos, int(f.n[0]), int(f.n[0]) + c)
            n, per = _take_counts(f, [c] * S, m)
            produced, handed = produced + k * S, handed + n
            assert k == (10, 690, 690)[i] and f.pool.pending() == produced - handed
            if not small_buffer:
                assert n == k * S and per == [k] * S
                assert i != 1 or n == cap                           # the push that fills the device buffer
                f.check()
            else:
                assert n == min(m, produced - handed + n)
                _check_prefix(f)
        if small_buffer:
            assert f.pool.pending() > cap
            f.take(f.pool.fetch(max_events=f.pool.pending()))
            assert f.pool.pending() == 0
            f.check()
    finally:
        f.close()


# Calibration push: n_len = 65 520 and max_chunk = 800, so c = n_len is what lets the push that completes calibration close
# its segments (E = ceil(829 / 19) = 44 against ceil(10 / 19) = 1 without c). The period-19 string cannot realise itself
# under its own noise_atap: with 9 loud blocks in 19 and a mean at mid_val, the quiet blocks carry as much |x - mid| as
# the loud ones, and a loud frame sums only 1.055 times the window's average frame (s_thl is 1.1 times it). So the window
# starts with 40 quiet blocks and holds 41 periods; loud samples sit 450 above mid_val and quiet ones 369 below it, which
# puts mid_val at exactly 2 048, n_thl between 369 and 450 (quiet samples in band, no low markers, so no crossing counts),
# and s_thl just under a loud frame's sum (160 * 450) and well above a mixed frame's (80 * 450 + 80 * 369).
CAL_LEN, CAL_CHUNK, CAL_LEAD = 65520, 800, 40
CAL_LOUD, CAL_QUIET = 2048 + 450, 2048 - 369


def calibration_stream(n_frames):
    """CAL_LEAD quiet blocks, then period-19 activity at CAL_LOUD / CAL_QUIET"""
    act = period_act(n_frames, CAL_LEAD)
    return np.where(plant_act(act) == LOUD, CAL_LOUD, CAL_QUIET).astype(np.uint16), act


def test_calibration_stream_realises_its_string_under_its_own_atap():
    """on the CPU: noise_atap over the first 65 520 samples gives mid_val 2 048 and thresholds under which the long-form
    VAD oracle finds exactly the string's segments, 41 of them closing in the calibration window's frames"""
    lo, port = ox.long_oracle(), ob.port()
    x, act = calibration_stream(900)
    at = port.noise_atap(np.ascontiguousarray(x[:CAL_LEN]), CAL_LEN)
    assert int(at["mid_val"][0]) == 2048 and 369 < int(at["n_thl"][0]) < 450, at
    assert 80 * (450 + 369) < int(at["s_thl"][0]) < 160 * 450, at
    n, seg = lo.vad_long(x[None, :], at, 128)
    assert [tuple(s) for s in seg[0, :int(n[0])].tolist()] == fsm_seq(act[:frames_of(len(x))])
    assert closings_between(period_closings(900, CAL_LEAD), 0, CAL_LEN + CAL_CHUNK - 1) == 41
    assert 41 > -(-(-(-CAL_CHUNK // 80)) // 19) == 1 and events_per_push(CAL_CHUNK, CAL_LEN) == 44


@pytest.mark.gpu
def test_event_buffer_at_the_calibration_push(handle, bank):
    """pushes of 799 samples: no frame is evaluated before n reaches 65 520; the push that completes calibration evaluates
    the 827 frames so far and closes 41 segments per stream, more than a bound without c allows; prefix equality after
    every push from then on"""
    handle.set_bank(bank[0], bank[1], 4096)
    S = 8
    x, _ = calibration_stream(1400)
    clos = period_closings(1400, CAL_LEAD)
    f = Feed(handle, [x] * S, CAL_CHUNK, CAL_LEN)
    try:
        assert f.pool.max_events == S * events_per_push(CAL_CHUNK, CAL_LEN) == S * 44
        cal_push = False
        while f.n[0] + 799 <= len(x) - 80:
            n0 = int(f.n[0])
            n, per = _take_counts(f, [799] * S)
            # no frame is evaluated before calibration completes; its push evaluates every frame so far
            want = closings_between(clos, n0 if n0 >= CAL_LEN else 0, n0 + 799) if n0 + 799 >= CAL_LEN else 0
            assert per == [want] * S, (n0, per, want)
            if n0 < CAL_LEN <= n0 + 799:
                assert want == 41 and n == 41 * S
                cal_push = True
            if n0 + 799 >= CAL_LEN:
                f.check()
        assert cal_push
    finally:
        f.close()
