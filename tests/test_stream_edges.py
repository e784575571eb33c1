"""The fixed-capture stream pool (sr_streams_* / sr_stream_group_*, K4 in csrc/sr_stream.cu) at its edges.

Every case is checked after EVERY push, not only at the end, against the CPU oracle on the full buffer:
  - an event arrives in the push that delivers sample max(end + 879, n_len - 1): the frame that closes a segment is
    evaluated once n >= end + 880, and nothing is evaluated before the calibration window is complete;
  - segments() is the oracle's VAD on the whole capture, masked: a start is shown once n >= start + 720 (long_fsm_window
    opens at frame start/80 + 7, frame k is evaluated once n >= 80k + 160) and an end once n >= end + 880; the reference FSM never
    abandons an opened segment, so a shown start is final;
  - atap is zero until the first n_len samples are in, then the oracle's noise_atap (zero for ever when n_len is 0 or not
    a multiple of 240: VAD.C:33-36 leaves it untouched);
  - every event equals get_mfcc (x[-1] = mid_val for a segment at sample 0, as every batched call), dtw with the save_sign
    check (or the banded DP under SR_DTW_BAND) and the strict-'<', first-wins argmin from (0, SR_DIS_MAX).
Events are compared per stream: within one push their order across streams follows the step kernel's atomic slots.

CPU: a header guard; the planted recordings of the GPU tests realise what they claim under the oracle (zero-atap runs of
exact lengths, a segment that opens only through last_sig carried over a 32-frame word edge).
GPU: capture lengths 161 ... 65 535 at every row alignment with lock-step chunks 1 ... 881 and ragged schedules (empty
pushes and pushes past the end included); calibration windows 0 ... 65 520 (scalar noise_atap_warp, catch-up pushes,
full-scale rows); last_sig carried across pushes cut around word edges; 119- and 120-frame segments in both geometries,
a fourth and fifth word, no bank and an all-unsigned bank; bursts of 6 144 events in one push (the second D2H copy) on a
pool, through fetch and on a group; the matcher, bank, DTW variant and geometry switched between pushes; reset with
events queued; groups of uneven shards with caller buffers of 0, 1 and 5 events drained by empty pushes."""
import os
import re

import numpy as np
import pytest

import oracle_bind as ob
import sr_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "golden.npz"))
NULL = 0xFFFFFFFF
ST_OK, ST_MFCC_FAIL = 0, 2
EV = ("stream", "segment", "start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")
REF, GEOM_B = 0, 1
GREEDY = (0, 0)


@pytest.fixture(scope="module")
def ora():
    return ob.best_oracle()


# ---- planted recordings (numpy only) -------------------------------------------------------------------------------------
def runs_pcm(L, runs, seed):
    """zeros with nonzero noise (1 ... 4095) on each [a, b) of `runs`. Under the zero atap (n_len 0 or not a multiple of 240)
    frame k is active iff it holds a nonzero sample, so a run [a, b) with a, b multiples of 80, a >= 80, at least 8 frames
    long and followed by >= 960 zeros is exactly the segment [a - 80, b + 80): frm_num (b - a)/80 + 1 in the reference
    geometry, (b - a)/80 in GEOM_B"""
    rng = np.random.default_rng(seed)
    x = np.zeros(L, np.uint16)
    for a, b in runs:
        x[a:b] = rng.integers(1, 4096, b - a)
    return x


def frames_for(geom, frm):
    """run length b - a whose segment has `frm` frames in geometry `geom`"""
    return 80 * (frm - 1) if geom == REF else 80 * frm


def run_list(a0, lengths, gap=1200):
    runs, a = [], a0
    for n in lengths:
        runs.append((a, a + n))
        a += n + gap
    return runs


CAL_M = 2048


def carry_pcm(L, f, h_frame, seed):
    """a segment that opens only through last_sig carried from one out-of-band sample `f - h_frame` frames earlier.
    Samples [0, 2400): noise whose deviations stay inside the band noise_atap derives from them (mid 2048, n_thl 100:
    the largest deviation, 100, lies only below mid, and m - 100 is not < b_thl). Then exact quiet at mid, one sample
    at mid + 150 (>= a_thl: last_sig = 2) in frame h_frame (h_frame < 0: none), and in frame f the samples
    mid - 150, mid + 150, mid - 150 at 80f + 100 ... 102: three band crossings when the carried class is 2, two otherwise
    (z_thl = 2). Frames f + 1 ... f + 7 are loud (frm_sum > s_thl) and frame f + 8 is quiet again, so 8 active frames
    in a row, and a segment [80f, 80f + 720), exist only with the carry."""
    rng = np.random.default_rng(seed)
    x = np.full(L, CAL_M, np.uint16)
    for w in range(10):
        win = np.array([CAL_M + 99] * 121 + [CAL_M - 99] * 118 + [CAL_M - 100], np.uint16)
        x[240 * w:240 * (w + 1)] = win[rng.permutation(240)]
    if h_frame >= 0:
        x[80 * h_frame + 120] = CAL_M + 150
    x[80 * f + 100:80 * f + 103] = (CAL_M - 150, CAL_M + 150, CAL_M - 150)
    x[80 * f + 160:80 * f + 640] = CAL_M + 400
    return x


def vad_py(x, atap, reset_every=None):
    """VAD.C:97-218 over the whole buffer, as sro_vad; reset_every = 32: last_sig reset at every 32-frame word edge (the
    transcription a step kernel that does not carry cin across activity words would be)"""
    mid, n_thl, s_thl, z_thl = (int(atap[k][0]) for k in ("mid_val", "n_thl", "s_thl", "z_thl"))
    a_thl, b_thl = mid + n_thl, mid - n_thl
    last = cur = front = back = nseg = 0
    seg = [NULL] * 6
    x = x.astype(np.int64)
    for k, i in enumerate(range(0, len(x) - 160, 80)):
        if reset_every and k % reset_every == 0:
            last = 0
        fr = x[i:i + 160]
        s = int(np.abs(fr - mid).sum())
        z = 0
        for h in range(159):
            v, w = fr[h], fr[h + 1]
            if v >= a_thl:
                last = 2
            elif v < b_thl:
                last = 1
            if w >= a_thl:
                z += last == 1
            elif w < b_thl:
                z += last == 2
        if s > s_thl or z > z_thl:
            if cur == 0:
                cur, front = 1, 1
            elif cur == 1:
                front += 1
                if front >= 8:
                    cur, front, seg[2 * nseg] = 2, 0, i - 560
            elif cur == 3:
                cur, back = 2, 0
        else:
            if cur == 2:
                cur, back = 3, 1
            elif cur == 3:
                back += 1
                if back >= 11:
                    cur, back, seg[2 * nseg + 1] = 0, 0, i - 880 + 160
                    nseg += 1
                    if nseg == 3:
                        break
            elif cur == 1:
                cur, front = 0, 0
    return seg


# ---- the oracle's view of a capture -------------------------------------------------------------------------------------
def oracle_capture(ora, pcm, n_len):
    """(atap [S], seg_off [S][3][2]) of the whole buffers: noise_atap of the first n_len samples on a zero atap, VAD over L"""
    S, L = pcm.shape
    atap = np.zeros(S, ob.ATAP_DTYPE)
    seg = np.zeros((S, 3, 2), np.uint32)
    for s in range(S):
        if n_len:                                   # n_len 0 leaves the zero atap (the reference would divide by zero)
            atap[s] = ora.noise_atap(pcm[s], n_len, atap[s:s + 1])[0]
        seg[s] = ora.vad(pcm[s], L, atap[s:s + 1]).reshape(3, 2)
    return atap, seg


def closed_keys(seg):
    return [(s, k) for s in range(seg.shape[0]) for k in range(3) if seg[s, k, 1] != NULL]


def oracle_events(ora, pcm, atap, seg, keys, geom=REF, match=GREEDY, bank=None, T=0):
    """{(stream, segment): event tuple} of `keys` under one setting: features on [mid_val, row...] rows (x[-1] of a
    segment at sample 0 is mid_val), dtw with the save_sign check or the banded DP, the strict-'<' first-wins argmin"""
    out = {}
    keys = list(keys)
    for c0 in range(0, len(keys), 128):
        part = keys[c0:c0 + 128]
        rows_s = np.array([s for s, _ in part])
        rows = ob.pinned_rows(pcm[rows_s], atap[rows_s])
        sg = np.array([seg[s, k] for s, k in part], np.uint32) + 1
        f = ob.port().mfcc_geom_b_batch(rows, sg, atap[rows_s]) if geom == GEOM_B else ora.mfcc_batch(rows, sg, atap[rows_s])
        ok = f["frm_num"] > 0
        idx = np.zeros(len(part), np.int64)
        dis = np.full(len(part), NULL, np.int64)
        if T and ok.any():
            if match[0] & sr_b200.DTW_BAND:
                sc, _ = ob.port().dtw_batch(f[ok], bank, T, 4096, check_sign=1, band_r=match[1])
            else:
                sc, _ = ora.dtw_batch(f[ok], bank, T, 4096, check_sign=1)
            key = (sc.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)
            kmin = key.min(axis=1)
            idx[ok] = (kmin & np.uint64(NULL)).astype(np.int64)
            dis[ok] = (kmin >> np.uint64(32)).astype(np.int64)
        for j, (s, k) in enumerate(part):
            fr = int(f["frm_num"][j])
            st = ST_OK if fr else ST_MFCC_FAIL
            bi, bd = (int(idx[j]), int(dis[j])) if fr else (0, NULL)
            out[(s, k)] = (s, k, int(seg[s, k, 0]), int(seg[s, k, 1]), st, fr, bi, bd, bi // 4)
    return out


def ev_tuple(e):
    return tuple(int(e[k]) for k in EV)


class Capture:
    """one capture pushed into a pool or group, checked after every push against the oracle's full-buffer result"""

    def __init__(self, pool, pcm, n_len, atap, seg):
        self.pool, self.pcm, self.n_len = pool, pcm, n_len
        self.S, self.L = pcm.shape
        self.atap, self.seg = atap, seg.astype(np.int64)
        self.cal_atap = n_len != 0 and n_len % 240 == 0
        self.pos = np.zeros(self.S, np.int64)
        self.events, self.pushes = [], 0
        self.push_of = {}

    def push(self, lens, lock=False, max_events=None, timing=True, poison=4095):
        S, L = self.S, self.L
        lens = np.asarray(lens, np.int64)
        w = int(lens.max()) if lens.size else 0
        chunk = np.full((S, w), poison, np.uint16)   # samples past L are dropped by the pool: poison them
        for s in range(S):
            take = max(0, min(int(lens[s]), L - int(self.pos[s])))
            chunk[s, :take] = self.pcm[s, self.pos[s]:self.pos[s] + take]
        if lock:
            evs = self.pool.push(chunk, max_events=max_events)
        else:
            evs = self.pool.push_ragged(chunk, lens, max_events=max_events)
        before = self.pos.copy()
        self.pos = np.minimum(self.pos + lens, L)
        for e in evs:
            s, k = e["stream"], e["segment"]
            assert (s, k) not in self.push_of, ("duplicate event", e)
            self.push_of[(s, k)] = self.pushes
            if timing:
                due = max(int(e["end"]) + 880, self.n_len)
                assert before[s] < due <= self.pos[s], (e, before[s], self.pos[s], self.n_len)
        self.events += evs
        self.pushes += 1
        self.check_state()
        return evs

    def check_state(self):
        seg, atap = self.pool.segments()
        n = self.pos
        cal = n >= self.n_len
        st, en = self.seg[:, :, 0], self.seg[:, :, 1]
        show_st = cal[:, None] & (st != NULL) & (n[:, None] >= st + 720)
        show_en = cal[:, None] & (en != NULL) & (n[:, None] >= en + 880)
        want = np.stack([np.where(show_st, st, NULL), np.where(show_en, en, NULL)], -1)
        assert np.array_equal(seg.astype(np.int64), want), (self.pushes, np.argwhere(seg.astype(np.int64) != want)[:4])
        wa = np.zeros(self.S, ob.ATAP_DTYPE)
        if self.cal_atap:
            wa[cal] = self.atap[cal]
        assert atap.tobytes() == wa.tobytes(), (self.pushes, np.nonzero(atap != wa)[0][:8])

    def check_events(self, want, complete=True):
        """every event equals `want` (a dict, or a callable of the push index), none twice; complete: every segment the
        oracle closes within the samples pushed came out"""
        got = {}
        for e in self.events:
            key = (e["stream"], e["segment"])
            w = want(self.push_of[key]) if callable(want) else want
            assert ev_tuple(e) == w[key], (ev_tuple(e), w[key])
            got[key] = e
        assert len(got) == len(self.events)
        if complete:
            due = [(s, k) for s, k in closed_keys(self.seg.astype(np.uint32))
                   if self.pos[s] >= max(self.seg[s, k, 1] + 880, self.n_len)]
            assert sorted(got) == sorted(due)
        return got


def lock_schedule(L, c, due):
    """chunks of c; 1-sample chunks cover 1 000 samples up to the first sample that closes an event (`due`), with the
    samples before and after in chunks of at most L"""
    if c >= 79 or L <= 2000:
        return [c] * (-(-L // c))
    a = max(0, min(due, L) - 800)
    out = [a] if a else []
    out += [1] * min(1000, L - a)
    rest = L - sum(out)
    return out + ([rest] if rest > 0 else [])


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_every_stream_pool_entry_point_is_run_here():
    """every sr_streams_* / sr_stream_group_* entry point of include/speech_recog.h is called by a GPU test of this file"""
    hdr = open(os.path.join(ROOT, "include", "speech_recog.h")).read()
    names = set(re.findall(r"\b(?:int|uint32_t)\s+(sr_(?:streams|stream_group)_\w+)\s*\(", hdr))
    # Capture pushes ragged unless lock=True, and calls segments() after every push
    py = {"sr_streams_create": "StreamPool(h,", "sr_streams_destroy": "pool.close()", "sr_streams_reset": "pool.reset()",
          "sr_streams_push": "pool.push(", "sr_streams_push_ragged": "Capture(pool,", "sr_streams_fetch": "pool.fetch(",
          "sr_streams_pending": "pool.pending()", "sr_streams_segments": "Capture(pool,",
          "sr_stream_group_create": "StreamPool(hs,", "sr_stream_group_destroy": "grp.close()",
          "sr_stream_group_reset": "grp.reset()", "sr_stream_group_push": "grp.push(",
          "sr_stream_group_push_ragged": "Capture(grp,", "sr_stream_group_segments": "Capture(grp,"}
    assert names == set(py), names
    src = open(os.path.abspath(__file__)).read()
    gpu = src[src.index("# ---- GPU"):]
    for n in names:
        assert gpu.count(py[n]) >= 1, n


@pytest.mark.parametrize("geom", [REF, GEOM_B])
def test_planted_runs_are_segments_of_the_planned_length(geom):
    """runs_pcm: under the zero atap the oracle's VAD finds [a - 80, b + 80) per run, with 119, 120 and 200 frames in the
    geometry's own framing; the first run, at a = 80, opens at sample 0; a fourth and fifth run are never reported"""
    po = ob.port()
    L = 65535
    lens = [frames_for(geom, 119), frames_for(geom, 120), frames_for(geom, 200), 640, 800]
    runs = run_list(80, lens)
    x = runs_pcm(L, runs, 1)
    atap = np.zeros(1, ob.ATAP_DTYPE)
    seg = po.vad(x, L, atap).reshape(3, 2)
    assert seg.tolist() == [[a - 80, b + 80] for a, b in runs[:3]] and seg[0, 0] == 0
    fl = 160 if geom == REF else 200
    assert [(e - s - fl) // 80 + 1 for s, e in seg.tolist()] == [119, 120, 200]
    # one nonzero sample anywhere makes its two frames active: a gap of 960 zeros is the least that closes a segment
    y = runs_pcm(12000, [(800, 1600), (2560, 3200)], 2)
    assert po.vad(y, 12000, atap).tolist()[:4] == [720, 1680, 2480, 3280]
    y = runs_pcm(12000, [(800, 1600), (2480, 3200)], 2)
    assert po.vad(y, 12000, atap).tolist()[:2] == [720, 3280]


def test_carried_last_sig_over_a_word_edge_opens_the_segment():
    """carry_pcm: the oracle opens [80f, 80f + 720) only when the out-of-band sample 40 frames earlier is carried; a VAD
    that resets last_sig at every 32-frame word edge loses the segment, and so does the capture without that sample"""
    po = ob.port()
    L, f = 12000, 80
    x = carry_pcm(L, f, 40, 3)
    atap = po.noise_atap(x, 2400)
    assert (int(atap["mid_val"][0]), int(atap["n_thl"][0]), int(atap["z_thl"][0])) == (CAL_M, 100, 2)
    assert 80 * 400 > int(atap["s_thl"][0]) > 160 * 100
    want = [80 * f, 80 * f + 720] + [NULL] * 4
    assert po.vad(x, L, atap).tolist() == want
    assert vad_py(x, atap) == want                                  # the transcription is faithful ...
    assert vad_py(x, atap, reset_every=32) == [NULL] * 6            # ... and loses the segment without the carry
    assert (f - 40) >= 33 and 40 // 32 != f // 32
    assert po.vad(carry_pcm(L, f, -1, 3), L, atap).tolist() == [NULL] * 6


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _handle(bank=None, T=0, geom=REF):
    h = sr_b200.Handle(0)
    if bank is not None:
        h.set_bank(bank, T, 4096)
    h.set_geometry(geom)
    return h


def _ragged(rng, S, L, choices, extra=2):
    """random per-stream lengths until every stream is full, then `extra` pushes past L; an all-zero push now and then"""
    pos, out = np.zeros(S, np.int64), []
    while (pos < L).any():
        lens = rng.choice(choices, S).astype(np.int64)
        if len(out) % 7 == 3:
            lens[:] = 0
        lens = np.minimum(lens, L)
        out.append(lens)
        pos += lens
    return out + [np.minimum(rng.choice(choices, S), L).astype(np.int64) for _ in range(extra)]


@pytest.mark.gpu
@pytest.mark.parametrize("L", [161, 239, 241, 8003, 8004, 39999, 65535])
def test_capture_lengths_at_every_row_alignment(ora, L):
    """S = 9 and 33 rows of L samples start at every 2-byte offset mod 16 (L odd, L = 4 mod 8): the scalar append, the
    unaligned block_scan and the (xb & 3) fallback around block_scan_split8. Lock-step chunks 1 ... 881, L at once, L - 1
    then 1, ragged schedules with empty pushes and pushes past L. L = 161 has one frame, 65 535 has 818"""
    bank, T = GOLD["synth/bank"], 8
    n_len = 2400 if L >= 2400 else (240 * (L // 240) if L >= 240 else 0)
    h = _handle(bank, T)
    for S in (9, 33):
        pcm = sr_b200.synth_pcm_host(S, L, 0x5E0000 + L + S, 3)
        if L >= 8000:
            pcm[2] = CAL_M                                              # a silent stream
        atap, seg = oracle_capture(ora, pcm, n_len)
        want = oracle_events(ora, pcm, atap, seg, closed_keys(seg), bank=bank, T=T)
        if L >= 8000:
            assert len(want) >= S - 1
        due = min([max(int(seg[s, k, 1]) + 880, n_len) for s, k in want] or [L // 2])
        scheds = [("lock", lock_schedule(L, c, due)) for c in (1, 79, 80, 81, 159, 160, 161, 879, 880, 881) if c <= L]
        scheds += [("lock", [L]), ("lock", [L - 1, 1])]
        rng = np.random.default_rng(L + S)
        scheds += [("ragged", _ragged(rng, S, L, [0, 1, 79, 80, 81, 160, 333, 880, 1601, 4000])) for _ in range(2)]
        pool = sr_b200.StreamPool(h, S, L, n_len)
        for i, (kind, sched) in enumerate(scheds):
            if i:
                pool.reset()
            cap = Capture(pool, pcm, n_len, atap, seg)
            for lens in sched:
                cap.push(np.full(S, lens, np.int64) if kind == "lock" else lens, lock=(kind == "lock"))
            assert (cap.pos == L).all()
            cap.check_events(want)
        pool.close()
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_len", [0, 160, 240, 2400, 2560, 2640, 4800, 64800, 65520, "L"])
def test_calibration_windows(ora, n_len):
    """n_len 0, 160 and 2 560 leave the zero atap (exact-zero runs open and close segments, one at sample 0); 2 640 is
    the first window the scalar noise_atap_warp sums; 64 800 and 65 520 make the calibration push a catch-up over ~810 blocks,
    and 65 520 sums full-scale rows to 4 293 853 200, just under 2^32; n_len = L = 24 000 calibrates on the whole
    capture. Stream S - 1 never receives n_len samples: no event, NULL segments, zero atap"""
    L = 24000 if n_len == "L" else 65535
    n_len = L if n_len == "L" else n_len
    S = 19
    bank, T = GOLD["synth/bank"], 8
    pcm = sr_b200.synth_pcm_host(S, L, 0xCA1000 + n_len, 3)
    rng = np.random.default_rng(n_len)
    for s in range(S):                                                   # exact-zero runs: silence under the zero atap
        for a in sorted(rng.choice(np.arange(20, L // 80 - 30), 4, replace=False)):
            pcm[s, 80 * a:80 * a + int(rng.integers(12, 30)) * 80] = 0
    pcm[1, :80] = 0
    pcm[1, 80:1600] = rng.integers(1, 4096, 1520)                        # zero atap: a segment at sample 0
    pcm[1, 1600:3000] = 0
    if n_len == 65520:
        pcm[3:6] = 0xFFFF                                                # full-scale rows
        pcm[4, 65520:] = 0
    atap, seg = oracle_capture(ora, pcm, n_len)
    if n_len % 240 or n_len == 0:
        assert (atap.view(np.uint8) == 0).all() and seg[1, 0, 0] == 0 and len(closed_keys(seg)) >= S
    h = _handle(bank, T)
    pool = sr_b200.StreamPool(h, S, L, n_len)
    want = oracle_events(ora, pcm, atap, seg, closed_keys(seg), bank=bank, T=T)
    short = max(n_len - 1, 0)
    for sched in ("ragged", "lock", "whole"):
        cap = Capture(pool, pcm, n_len, atap, seg)
        if sched == "ragged":
            r = np.random.default_rng(n_len + 1)
            for lens in _ragged(r, S, L, [0, 1, 80, 81, 333, 2399, 2401, 4000, 20000]):
                lens[S - 1] = min(lens[S - 1], max(short - cap.pos[S - 1], 0))   # stream S - 1 stops short of n_len
                cap.push(lens)
        elif sched == "lock":
            for _ in range(-(-L // 4001)):
                cap.push(np.full(S, 4001), lock=True)
        else:
            cap.push(np.full(S, L), lock=True)
        if sched == "ragged" and n_len:
            assert cap.pos[S - 1] == short
            assert not any(e["stream"] == S - 1 for e in cap.events)
        cap.check_events(want)
        pool.reset()
    pool.close()
    h.close()


@pytest.mark.gpu
def test_carried_last_sig_across_pushes_and_word_edges(ora):
    """carry_pcm pushed with boundaries one block before and after each 32-frame word edge (of the samples and of the
    frames they complete), in 80-sample chunks and whole: the segment that exists only through the carried class opens
    and closes as the oracle says. Streams differ in the distance to the carried sample (33 ... 70 frames) and one has
    none"""
    L, S = 12000, 8
    fs = [80, 90, 100, 110, 112, 120, 97, 80]
    hs = [40, 57, 30, 70, 79, 50, 31, -1]
    pcm = np.stack([carry_pcm(L, f, hf, 3 + s) for s, (f, hf) in enumerate(zip(fs, hs))])
    atap, seg = oracle_capture(ora, pcm, 2400)
    assert [tuple(seg[s, 0]) for s in range(S)] == [(80 * f, 80 * f + 720) for f in fs[:-1]] + [(NULL, NULL)]
    assert all(f - hf >= 33 and f // 32 != hf // 32 for f, hf in zip(fs[:-1], hs[:-1]))
    bank, T = GOLD["synth/bank"], 8
    want = oracle_events(ora, pcm, atap, seg, closed_keys(seg), bank=bank, T=T)
    h = _handle(bank, T)
    pool = sr_b200.StreamPool(h, S, L, 2400)
    cuts = sorted({80 * (32 * j + d) for j in range(1, 5) for d in (-1, 1, 2, 3)} | {2400})
    scheds = [np.diff([0] + cuts + [L]).tolist(), [80] * (L // 80), [L]]
    for i, sched in enumerate(scheds):
        if i:
            pool.reset()
        cap = Capture(pool, pcm, 2400, atap, seg)
        for c in sched:
            cap.push(np.full(S, c), lock=True)
        assert len(cap.check_events(want)) == S - 1
    pool.close()
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [REF, GEOM_B])
def test_failed_and_unmatched_events(ora, geom):
    """zero-atap runs whose segments have 119 frames (OK), 120 (SR_ST_MFCC_FAIL: frm_num 0, best_idx 0, best_dis
    0xFFFFFFFF, cmd 0) and 200 in the handle's geometry; a stream with five words reports three. Then the same on a
    handle without a bank and on a bank whose slots are all unsigned: every OK event carries the argmin initialiser"""
    L, S = 65535, 6
    f119, f120, f200 = (frames_for(geom, n) for n in (119, 120, 200))
    plans = [[f119, f120, f200], [f120, f119, 800], [f200, f119, f120], [640, 800, 960, 720, 880], [f120], [f119, 640]]
    pcm = np.stack([runs_pcm(L, run_list(80 + 80 * (s % 3), p), 10 + s) for s, p in enumerate(plans)])
    atap, seg = oracle_capture(ora, pcm, 0)
    keys = closed_keys(seg)
    assert len(keys) == 3 + 3 + 3 + 3 + 1 + 2 and seg[0, 0, 0] == 0
    bank, T = GOLD["synth/bank"], 8
    unsigned = bank.copy()
    unsigned[:, :2] = 0xFF
    for label, b, t in (("bank", bank, T), ("no bank", None, 0), ("unsigned", unsigned, T)):
        want = oracle_events(ora, pcm, atap, seg, keys, geom=geom, bank=b, T=t)
        fails = [k for k, w in want.items() if w[4] == ST_MFCC_FAIL]
        assert len(fails) == 6 and all(want[k][5:] == (0, 0, NULL, 0) for k in fails)
        if label != "bank":
            assert all(w[6:] == (0, NULL, 0) for w in want.values())
        h = _handle(b, t, geom)
        pool = sr_b200.StreamPool(h, S, L, 0)
        cap = Capture(pool, pcm, 0, atap, seg)
        for lens in _ragged(np.random.default_rng(geom), S, L, [0, 81, 960, 4001, 9999]):
            cap.push(lens)
        got = cap.check_events(want)
        assert len(got) == 15 and sum(1 for s, _ in got if s == 3) == 3
        pool.close()
        h.close()


def _burst_pcm(S, L, seed):
    rng = np.random.default_rng(seed)
    j = rng.integers(0, 8, (S, 3))
    pcm = np.zeros((S, L), np.uint16)
    for s in range(S):
        runs = [(80 * (1 + j[s, 0]), 80 * (1 + j[s, 0]) + 800), (2600 + 80 * j[s, 1], 3400 + 80 * j[s, 1]),
                (5000 + 80 * j[s, 2], 5800 + 80 * j[s, 2])]
        for a, b in runs:
            pcm[s, a:b] = rng.integers(1, 4096, b - a)
    return pcm


def _check_burst(h, ora, pcm, events, bank, T):
    """every event against the GPU batch calls (noise_atap, vad, mfcc + dtw per segment, recognise for segment 0), and
    64 of them against the oracle"""
    S, L = pcm.shape
    atap = h.noise_atap(pcm, 0)
    seg = h.vad(pcm, atap)
    assert (atap.view(np.uint8) == 0).all() and (seg[:, :, 1] != NULL).all()
    batch = {}
    for k in range(3):
        f = h.mfcc(pcm, seg[:, k, :], atap)
        _, bi, bd = h.dtw(f, flags=sr_b200.DTW_CHECK_SIGN)
        for s in range(S):
            batch[(s, k)] = (s, k, int(seg[s, k, 0]), int(seg[s, k, 1]), ST_OK, int(f["frm_num"][s]), int(bi[s]), int(bd[s]),
                             int(bi[s]) // 4)
    rec = h.recognise(pcm, 0, want=("best_idx", "best_dis", "status"))
    assert (rec["status"] == 0).all()
    got = {(e["stream"], e["segment"]): ev_tuple(e) for e in events}
    assert len(got) == len(events) == 3 * S and got == batch
    assert all((got[(s, 0)][6], got[(s, 0)][7]) == (int(rec["best_idx"][s]), int(rec["best_dis"][s])) for s in range(S))
    sample = sorted(np.random.default_rng(S).choice(len(got), 64, replace=False).tolist())
    keys = [sorted(got)[i] for i in sample]
    want = oracle_events(ora, pcm, atap, seg, keys, bank=bank, T=T)
    assert all(got[k] == want[k] for k in keys)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["default_buffer", "fetch", "group"])
def test_burst_past_the_quick_window(ora, mode):
    """S = 2 048 streams close three words each in one whole-capture push: 6 144 events, more than StreamCore::kQuick =
    4 096, so the push makes its second D2H copy. With the default buffer all come back at once; with max_events = 4 000
    the rest is queued and fetched; a group of two handles on one device (S = 4 096) crosses the window in each shard"""
    L = 8000
    S = 4096 if mode == "group" else 2048
    bank, T = GOLD["synth/bank"], 8
    pcm = _burst_pcm(S, L, 0xB0057 + S)
    hs = [_handle(bank, T) for _ in range(2 if mode == "group" else 1)]
    if mode == "group":
        grp = sr_b200.StreamPool(hs, S, L, 0)
        events = grp.push(pcm)
        grp.close()
    else:
        pool = sr_b200.StreamPool(hs[0], S, L, 0)
        if mode == "fetch":
            events = pool.push(pcm, max_events=4000)
            assert len(events) == 4000 and pool.pending() == 3 * S - 4000
            events += pool.fetch()
            assert pool.pending() == 0
        else:
            events = pool.push(pcm)
        pool.close()
    assert len(events) == 3 * S > 4096
    _check_burst(hs[0], ora, pcm, events, bank, T)
    for h in hs:
        h.close()


@pytest.mark.gpu
def test_settings_switched_between_pushes(ora):
    """during one capture the matcher (greedy, band r = 0, 7, 118), the bank (sr_set_bank to another bank, then
    sr_set_bank_dev), the DTW variant and the geometry change before pushes: every event equals the oracle under the
    settings in force at the push that emitted it"""
    import torch
    S, L = 24, 40000
    pcm = sr_b200.synth_pcm_host(S, L, 0x5E77, 3)
    atap, seg = oracle_capture(ora, pcm, 2400)
    keys = closed_keys(seg)
    assert len(keys) >= 2 * S
    fb = sr_b200.synth_ftr_host(11, 0xB4, 20, 119).view(sr_b200.FTR_DTYPE).reshape(-1)
    fc = sr_b200.synth_ftr_host(5, 0xC4, 30, 90).view(sr_b200.FTR_DTYPE).reshape(-1)
    banks = {"A": (GOLD["synth/bank"], 8), "B": (sr_b200.make_bank(fb, valid=np.arange(11) % 3 != 1), 11),
             "C": (sr_b200.make_bank(fc), 5)}
    bank_c = torch.from_numpy(banks["C"][0]).to("cuda:0")
    # (geometry, matcher, bank, dtw variant)
    plan = [(REF, GREEDY, "A", 0), (REF, (sr_b200.DTW_BAND, 0), "A", 0), (REF, (sr_b200.DTW_BAND, 7), "B", 0),
            (GEOM_B, (sr_b200.DTW_BAND, 118), "B", 1), (GEOM_B, GREEDY, "C", 1), (REF, GREEDY, "C", 0),
            (GEOM_B, (sr_b200.DTW_BAND, 7), "A", 1), (REF, (sr_b200.DTW_BAND, 118), "C", 0)]
    h = sr_b200.Handle(0)
    pool = sr_b200.StreamPool(h, S, L, 2400)
    cap = Capture(pool, pcm, 2400, atap, seg)
    used = []
    for i in range(L // 800):
        geom, match, b, var = plan[i % len(plan)]
        h.set_geometry(geom)
        h.set_match(*match)
        if b == "C":
            h.set_bank_dev(bank_c.data_ptr(), banks["C"][1], 4096)
        else:
            h.set_bank(*banks[b], 4096)
        h.set_dtw_variant(var)
        used.append(i % len(plan))
        cap.push(np.full(S, 800), lock=True)
    torch.cuda.synchronize()
    by_setting = {}
    for (s, k), p in cap.push_of.items():
        by_setting.setdefault(used[p], []).append((s, k))
    want = {}
    for j, ks in by_setting.items():
        geom, match, b, _ = plan[j]
        want.update(oracle_events(ora, pcm, atap, seg, ks, geom=geom, match=match, bank=banks[b][0], T=banks[b][1]))
    cap.check_events(want)
    assert len(by_setting) >= 4
    pool.close()
    h.close()


def _sorted_events(evs):
    return sorted(ev_tuple(e) for e in evs)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pool", "group"])
def test_reset_with_queued_events_then_different_audio(ora, kind):
    """reset() mid-capture while events are queued (every push returned none): the queue is dropped (pending() is 0 on a
    pool; on a group an empty push returns nothing), and the next capture of different audio gives exactly what a fresh
    pool gives, and the oracle"""
    S, L = 24, 16000
    bank, T = GOLD["synth/bank"], 8
    a = sr_b200.synth_pcm_host(S, L, 0xA0A0, 3)
    b = sr_b200.synth_pcm_host(S, L, 0xB0B0, 3)
    atap, seg = oracle_capture(ora, b, 2400)
    want = oracle_events(ora, b, atap, seg, closed_keys(seg), bank=bank, T=T)
    hs = [_handle(bank, T) for _ in range(2)]
    results = []
    for fresh in (False, True):
        if kind == "pool":
            pool = sr_b200.StreamPool(hs[0], S, L, 2400)
            obj = pool
        else:
            grp = sr_b200.StreamPool(hs, S, L, 2400)
            obj = grp
        if not fresh:
            for n0 in (0, 4000, 8000):
                assert obj.push(np.ascontiguousarray(a[:, n0:n0 + 4000]), max_events=0) == []
            if kind == "pool":
                assert pool.pending() > 0
                pool.reset()
                assert pool.pending() == 0
            else:
                grp.reset()
                assert grp.push(np.zeros((S, 0), np.uint16)) == []
        cap = Capture(pool if kind == "pool" else grp, b, 2400, atap, seg)
        for lens in _ragged(np.random.default_rng(9), S, L, [0, 80, 333, 1601, 4000]):
            cap.push(lens)
        cap.check_events(want)
        results.append((_sorted_events(cap.events), cap.pool.segments()[0].tobytes()))
        if kind == "pool":
            pool.close()
        else:
            grp.close()
    assert results[0] == results[1]
    for h in hs:
        h.close()


@pytest.mark.gpu
def test_group_uneven_shards_small_buffers_drained_by_empty_pushes(ora):
    """S = 37 over three handles on one device (shards of 12, 12 and 13 streams), ragged pushes that hand out at most 0,
    1 or 5 events each, then empty pushes until the queue is dry: nothing lost or duplicated, global stream numbers, each
    stream's events in segment order, segments() equal to the oracle's. pending() and fetch() refuse a group"""
    S, L = 37, 16000
    bank, T = GOLD["synth/bank"], 8
    pcm = sr_b200.synth_pcm_host(S, L, 0x37, 3)
    atap, seg = oracle_capture(ora, pcm, 2400)
    want = oracle_events(ora, pcm, atap, seg, closed_keys(seg), bank=bank, T=T)
    assert len(want) >= 2 * S
    hs = [_handle(bank, T) for _ in range(3)]
    grp = sr_b200.StreamPool(hs, S, L, 2400)
    with pytest.raises(sr_b200.SrError):
        grp.pending()
    with pytest.raises(sr_b200.SrError):
        grp.fetch()
    cap = Capture(grp, pcm, 2400, atap, seg)
    sched = _ragged(np.random.default_rng(37), S, L, [0, 1, 79, 81, 1601, 4000, 8000])
    for i, lens in enumerate(sched):
        evs = cap.push(lens, max_events=(0, 1, 5)[i % 3], timing=False)
        assert len(evs) <= (0, 1, 5)[i % 3]
    assert (cap.pos == L).all() and len(cap.events) < len(want)
    drains = 0
    while True:
        evs = grp.push(np.zeros((S, 0), np.uint16), max_events=5)
        for e in evs:
            cap.push_of[(e["stream"], e["segment"])] = cap.pushes
        cap.events += evs
        drains += 1
        if not evs:
            break
        assert drains <= len(want)
    assert drains > 1
    cap.check_events(want)
    order = {}
    for e in cap.events:
        order.setdefault(e["stream"], []).append(e["segment"])
    assert all(v == list(range(len(v))) for v in order.values())
    assert max(order) >= 25                                            # the third shard's numbers are global
    cap.check_state()
    grp.close()
    for h in hs:
        h.close()
