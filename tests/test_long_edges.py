"""The long-form VAD where it carries state and splits work (csrc/sr_vad_long.cu): the 1 024-frame window edges of the
segment pass (K12), the work items of the block pass (K11b) and the flat segment table of recognition.

K12 walks each recording in windows of 1 024 frames and hands three things across every window edge: whether a segment is
open, the length of the run the FSM is counting there (fewer than 8 active or 11 inactive frames) and last_sig (`cin`).
Random speech leaves where edges fall relative to runs to chance, so the inputs here are planted: any frame-activity
string becomes PCM whose frame k is active exactly when the string says so (`plant`). Under PLANT_ATAP every sample is in
band except one priming sample at position 0 and one sample at 80(k+1) per active frame k, alternately above and below
the band. Sample 80(k+1) lies only in frame k's crossing window [80k+1, 80k+159], and it crosses because its class differs
from the previous out-of-band sample's, which may lie any number of windows earlier: a sparse string tests the carried
`cin` directly.

CPU: the planted PCM realises its string under the oracle (sro_vad_long) and the plain transcription of VAD.C; a Python
restatement of long_fsm_window equals the sequential FSM exhaustively on short strings; and the case table below reaches
every carried state at an edge with every way of completing or breaking it (asserted, so a case cannot silently go).
GPU (bit for bit against the oracle): the case table with its edge at windows 1, 2 and 7, through both VAD calls and
recognition; K11b's grid strides, short last items at both staging parities, skipped empty items; batch sizes on both
sides of the segment kernel's 8 recordings per CTA and the prefix kernel's 1 024 per pass."""
import itertools

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200

NULL = 0xFFFFFFFF
WIN = 1024                                  # frames per K12 window
PLANT_ATAP = (2048, 100, 0, 0xFFFFFFFF)     # mid, n_thl, z_thl, s_thl: a frame is active on one band crossing
EDGES = (1, 2, 7)                           # the window edge under test, in windows
MAX_SEGS = 6                                # the cut of the edge-table calls


# ---- planted inputs ------------------------------------------------------------------------------------------------------
def frames_of(n):
    """frames i = 80k while i < n - 160 (VAD.C:121)"""
    return -(-(n - 160) // 80) if n > 160 else 0


def plant(act, n=None):
    """PCM of n samples (default 80 N + 160) whose N = len(act) frames are active exactly where act is 1 under PLANT_ATAP"""
    act = np.asarray(act, np.uint8)
    n = 80 * len(act) + 160 if n is None else n
    assert frames_of(n) == len(act)
    pcm = np.full(n, 2048, np.uint16)
    pcm[0] = 1947                                           # below the band: last_sig = 1 before frame 0
    k = np.flatnonzero(act)
    pcm[80 * (k + 1)] = np.where(np.arange(len(k)) % 2 == 0, 2148, 1947)
    return pcm


def plant_atap(B):
    a = np.zeros(B, ob.ATAP_DTYPE)
    a["mid_val"], a["n_thl"], a["z_thl"], a["s_thl"] = PLANT_ATAP
    return a


def fsm_trace(act):
    """the sequential FSM of VAD.C:164-216 over an activity string: (segments [(start, end)], states {edge frame: (open,
    run, closed segments)} at every multiple of WIN, events [(open?, frame of the 8th / 11th frame, segment index)])"""
    cur = front = back = 0
    segs, states, events = [], {}, []
    for k, a in enumerate(act):
        if k and k % WIN == 0:
            states[k] = (cur >= 2, front if cur == 1 else back if cur == 3 else 0, len(segs) - (cur >= 2))
        if a:
            if cur == 0:
                cur, front = 1, 1
            elif cur == 1:
                front += 1
                if front >= 8:
                    cur, front = 2, 0
                    segs.append([80 * (k - 7), NULL])
                    events.append((True, k, len(segs) - 1))
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
                    events.append((False, k, len(segs) - 1))
            elif cur == 1:
                front, cur = 0, 0
    return [tuple(s) for s in segs], states, events


def fsm(act):
    return fsm_trace(act)[0]


def fsm_windowed(act, W):
    """long_fsm_window restated over windows of W frames: a run carried into a window completes at its first frames (need
    = 8 or 11 minus the carried run), later events are found inside the window only, and the run at the window's end
    (frames since the last breaking frame and since the last event) is carried on.

    In the kernel W is 1 024 and only the last window is shorter, so only the last window can be shorter than `need`
    (at most 11): the model is checked at W >= 11, and the short last windows are GPU cases of the edge table."""
    op, run, segs = False, 0, []

    def event(frame):
        if op:
            segs[-1][1] = 80 * frame + 80
        else:
            segs.append([80 * frame, NULL])
    for base in range(0, len(act), W):
        a = list(act[base:base + W])
        nw, cur, ev = len(a), 0, False
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


# ---- the edge table ------------------------------------------------------------------------------------------------------
def _runs(rng, n, lo=1, hi=14):
    """a run-structured activity string of n frames"""
    out, a = [], int(rng.integers(0, 2))
    while len(out) < n:
        out += [a] * int(rng.integers(lo, hi))
        a ^= 1
    return out[:n]


def _with_state(rng, e, op, r, nseg=0, head=True):
    """frames [0, e): a random head (or none), 20 inactive frames (closed, no run), nseg segments of 9 active + 12
    inactive frames, then the state at e: open with a run of r inactive frames, or closed with a run of r active ones"""
    ctl = 20 + 21 * nseg + 45
    act = np.zeros(e, np.uint8)
    if head:
        act[:e - ctl] = _runs(rng, e - ctl)
    p = e - ctl + 20
    for _ in range(nseg):
        act[p:p + 9] = 1
        p += 21
    if op:
        act[e - r - 30:e - r] = 1
    else:
        act[e - r:e] = 1
    return act


def _after(rng, op, j, brk, tail):
    """j frames that continue the run at the edge (inactive when open), one that breaks it if brk, then a random tail"""
    want = 0 if op else 1
    return np.r_[np.full(j, want, np.uint8), np.full(1 if brk else 0, 1 - want, np.uint8), _runs(rng, tail)].astype(np.uint8)


def edge_cases(w, seed=0):
    """[(name, activity)] with the window edge under test at frame e = WIN * w"""
    rng = np.random.default_rng(seed + w)
    e = WIN * w
    tails = (40, 120) if w >= 7 else (40, 300, 1500)
    out = []
    for op in (False, True):
        for r in range(11 if op else 8):
            need = (11 if op else 8) - r
            for j in range(need + 1):                           # j == need: the run completes; else it breaks after j
                act = np.r_[_with_state(rng, e, op, r), _after(rng, op, j, j < need, int(rng.choice(tails)))]
                out.append(("%s r%d %s" % ("open" if op else "closed", r, "complete" if j == need else "break%d" % j), act))
    # short last windows: nfr % WIN in 1..11, the carried run completes in it, breaks in it or neither
    for op, r in ((False, 3), (False, 7), (True, 2), (True, 10)):
        need = (11 if op else 8) - r
        plans = [(need, need, False), (min(11, need + 2), need, False),     # (L, j, brk): completes in it
                 (1, 0, True), (need, need - 1, True)]                        # breaks in it
        if need > 1:
            plans.append((need - 1, need - 1, False))                        # neither: it ends first
        for L, j, brk in plans:
            act = np.r_[_with_state(rng, e, op, r), _after(rng, op, j, brk, L - j - brk)]
            out.append(("%s r%d short last window %d" % ("open" if op else "closed", r, L), act))
    # events at the last frame of a window: an opening's 8th active frame, a closing's 11th inactive one
    act = _with_state(rng, e, False, 0)
    act[e - 8:e] = 1
    act[e - 9] = 0
    out.append(("opens at frame e-1", np.r_[act, _runs(rng, 60)]))
    out.append(("closes at frame e-1", np.r_[_with_state(rng, e, True, 11), _runs(rng, 60)]))
    # segments that open in one window and close two windows later (active runs with gaps of < 11 inactive frames)
    if w < 7:
        for k in range(2):
            act = _with_state(rng, e, False, 0)
            s = e - 300 - 100 * k
            long_seg = np.r_[np.ones(8, np.uint8), _runs(rng, WIN + 800 + s % 97, 1, 10), np.zeros(20, np.uint8)]
            out.append(("long segment %d" % k, np.r_[act[:s], np.zeros(20, np.uint8), long_seg, _runs(rng, 50)]))
    # max_segs cuts: segment MAX_SEGS - 1 (the last one written) or MAX_SEGS (the first not written) open at the edge, or
    # opened by a carried run
    for nseg in (MAX_SEGS - 1, MAX_SEGS):
        out.append(("cut %d open at the edge" % nseg,
                    np.r_[_with_state(rng, e, True, 4, nseg, head=False), _after(rng, True, 7, False, 60)]))
        out.append(("cut %d opened by a carried run" % nseg,
                    np.r_[_with_state(rng, e, False, 5, nseg, head=False), _after(rng, False, 3, False, 60)]))
    return out


def sparse_cases():
    """active frames 1 025 and 2 049+ frames apart, windows without one out-of-band sample, and 8-frame runs whose first
    frame is the first crossing after such a gap (one after a 7-frame run, one across an edge)"""
    out = []
    act = np.zeros(6 * WIN + 50, np.uint8)
    act[[5, 5 + 1025, 5 + 1025 + 2049, 5 + 1025 + 2049 + 2100]] = 1
    act[-30:-22] = 1
    out.append(("isolated frames", act))
    act = np.zeros(5 * WIN + 40, np.uint8)
    act[100:107] = 1                                        # 7 active frames: no segment
    act[107 + 1100:107 + 1108] = 1                          # the next crossing 1 100 frames later opens one
    act[3 * WIN - 3:3 * WIN + 5] = 1                        # the next, across an edge
    act[5 * WIN + 2:5 * WIN + 10] = 1
    out.append(("7 frames, a gap, 8 frames", act))
    act = np.zeros(8 * WIN, np.uint8)
    act[WIN - 1] = 1
    act[4 * WIN:4 * WIN + 8] = 1                            # 3 073 frames after the last crossing, at an edge
    act[8 * WIN - 8:] = 1
    out.append(("gap of three windows", act))
    return out


def random_cases(seed, n):
    rng = np.random.default_rng(seed)
    return [("random %d" % i, np.asarray(_runs(rng, int(rng.integers(2 * WIN, 8 * WIN))), np.uint8)) for i in range(n)]


# ---- coverage of the table -------------------------------------------------------------------------------------------------
def _outcome(act, e, op, r):
    need, want = (11 if op else 8) - r, 0 if op else 1
    j = 0
    while j < need and e + j < len(act) and act[e + j] == want:
        j += 1
    return "complete" if j == need else ("break", j) if e + j < len(act) else ("end", j)


def coverage(cases):
    """the rows of the edge table that `cases` reach"""
    got = set()
    for _, act in cases:
        _, states, events = fsm_trace(act)
        n = len(act)
        for e, (op, r, nclosed) in states.items():
            o = _outcome(act, e, op, r)
            got.add((op, r, o if o == "complete" else o[0] + str(o[1])))
            if n - e <= 11 and e == WIN * ((n - 1) // WIN) and r:
                got.add(("short", op, o if o == "complete" else o[0]))
            if op and nclosed in (MAX_SEGS - 1, MAX_SEGS):
                got.add(("cut open at edge", nclosed))
        for op, k, i in events:
            if k % WIN in (WIN - 1, 0) and k:
                got.add(("event at", op, k % WIN))
            if op and i in (MAX_SEGS - 1, MAX_SEGS) and k - 7 < WIN * (k // WIN):
                got.add(("cut opened by a carried run", i))
        opens = {i: k for op, k, i in events if op}
        for op, k, i in events:
            if not op and k // WIN >= opens[i] // WIN + 2:
                got.add("long segment")
        on = np.flatnonzero(act)
        gaps = np.diff(on)
        if len(gaps) and gaps.max() > WIN:
            got.add("gap > 1 window")
            if gaps.max() > 2 * WIN:
                got.add("gap > 2 windows")
            for op, k, i in events:
                if op and k - 7 in on[1:][gaps > WIN]:
                    got.add("opening after a gap")
        if any(not act[WIN * w:WIN * (w + 1)].any() for w in range(n // WIN)):
            got.add("window without a crossing")
    return got


def required_rows():
    rows = set()
    for op in (False, True):
        for r in range(11 if op else 8):
            rows.add((op, r, "complete"))
            rows |= {(op, r, "break%d" % j) for j in range((11 if op else 8) - r)}
        rows |= {("short", op, k) for k in ("complete", "break", "end")}
        rows |= {("event at", op, f) for f in (WIN - 1, 0)}
    rows |= {("cut open at edge", MAX_SEGS - 1), ("cut open at edge", MAX_SEGS), ("cut opened by a carried run", MAX_SEGS - 1),
             ("cut opened by a carried run", MAX_SEGS)}
    return rows | {"long segment", "gap > 1 window", "gap > 2 windows", "opening after a gap", "window without a crossing"}


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
def _oracle_segs(lo, acts, max_segs=4096):
    n = max(80 * len(a) + 160 for a in acts)
    pcm = np.full((len(acts), n), 2048, np.uint16)
    lens = np.zeros(len(acts), np.uint32)
    for b, a in enumerate(acts):
        p = plant(a)
        pcm[b, :len(p)] = p
        lens[b] = len(p)
    cnt, seg = lo.vad_long(pcm, plant_atap(len(acts)), max_segs, lens)
    return [[tuple(s) for s in seg[b, :min(int(cnt[b]), max_segs)].tolist()] for b in range(len(acts))], cnt


def test_planted_pcm_realises_its_activity_string():
    """sro_vad_long on the planted PCM equals the sequential FSM on the string: random and run-structured strings, the
    whole edge table; on short strings also the plain transcription of VAD.C (test_long.py)"""
    from test_long import py_vad_long
    lo = ox.long_oracle()
    rng = np.random.default_rng(0xED6E)
    acts = [rng.integers(0, 2, int(rng.integers(0, 400))).astype(np.uint8) for _ in range(100)]
    acts += [np.asarray(_runs(rng, int(rng.integers(1, 3000))), np.uint8) for _ in range(100)]
    acts += [a for w in EDGES for _, a in edge_cases(w)] + [a for _, a in sparse_cases()]
    got, cnt = _oracle_segs(lo, acts)
    for b, a in enumerate(acts):
        want = fsm(a)
        assert int(cnt[b]) == len(want) and got[b] == want, b
    assert sum(len(fsm(a)) for a in acts) > 1000
    for a in acts[:40]:
        assert py_vad_long(plant(a), 80 * len(a) + 160, plant_atap(1)[0]) == fsm(a)


@pytest.mark.parametrize("W", [11, 12])
def test_windowed_model_equals_sequential_fsm_exhaustively(W):
    """every activity string of up to 17 frames"""
    for L in range(1, 18):
        for s in itertools.product((0, 1), repeat=L):
            assert fsm_windowed(s, W) == fsm(s), (W, s)


def test_windowed_model_equals_sequential_fsm_on_runs():
    """run-structured strings over many edges, at window sizes 11 to 39 and the kernel's 1 024"""
    rng = np.random.default_rng(0x3F5)
    for t in range(600):
        W = int(rng.integers(11, 40))
        s = _runs(rng, int(rng.integers(1, 12 * W)), 1, int(rng.integers(3, 16)))
        assert fsm_windowed(s, W) == fsm(s), (W, s)
    for _, a in edge_cases(1)[::7] + sparse_cases():
        assert fsm_windowed(a.tolist(), WIN) == fsm(a)


def test_edge_table_reaches_every_row():
    """closed with run 0-7 and open with run 0-10 at an edge, each completed at `need` and broken after every earlier
    frame, at every edge position; short last windows; events at frames 1 023 / 1 024; long segments; max_segs cuts at an
    edge; sparse strings"""
    for w in EDGES:
        cases = edge_cases(w)
        got = coverage(cases)
        table = {r for r in required_rows() if isinstance(r, tuple) and r[0] in (False, True)}
        assert table <= got, (w, sorted(table - got, key=str))
        assert all(2 * WIN <= len(a) + WIN <= 9 * WIN for _, a in cases), w
    got = set().union(*(coverage(c) for c in [edge_cases(w) for w in EDGES] + [sparse_cases()]))
    missing = required_rows() - got
    assert not missing, sorted(missing, key=str)


# ---- GPU: window edges ------------------------------------------------------------------------------------------------------
def _batch(acts, U=None):
    """planted recordings in rows of U samples (default: the longest), poisoned past their length with loud band
    crossings"""
    lens = np.array([80 * len(a) + 160 for a in acts], np.uint32)
    U = int(lens.max()) if U is None else U
    pcm = np.empty((len(acts), U), np.uint16)
    for b, a in enumerate(acts):
        pcm[b, :lens[b]] = plant(a)
        pcm[b, lens[b]:] = np.where(np.arange(U - lens[b]) % 2, 4095, 0)
    return pcm, lens


def _check(names, got_n, got_seg, want_n, want_seg, what):
    bad = [names[b] for b in range(len(names)) if got_n[b] != want_n[b] or not np.array_equal(got_seg[b], want_seg[b])]
    assert not bad, "%s: %d rows differ, first %s" % (what, len(bad), bad[:5])


def _vad_dev(h, pcm, lens, max_segs, off=0, atap=None):
    """sr_vad_long_batch_dev on a copy of pcm at `off` bytes past a 16-byte boundary: (n_segs, seg_off) on the host"""
    import torch
    B, U = pcm.shape
    dev = torch.device("cuda:0")
    raw = torch.zeros(pcm.nbytes + 64, dtype=torch.uint8, device=dev)
    base = (16 - raw.data_ptr() % 16) % 16 + off
    raw[base:base + pcm.nbytes] = torch.from_numpy(pcm.view(np.uint8).reshape(-1)).to(dev)
    d_lens = torch.from_numpy(lens.view(np.int32)).to(dev)
    at = plant_atap(B) if atap is None else atap
    d_atap = torch.from_numpy(at.view(np.uint8).copy()).to(dev)
    d_n = torch.zeros(B, dtype=torch.int32, device=dev)
    d_seg = torch.zeros(B * max(max_segs, 1) * 2, dtype=torch.int32, device=dev)
    h.vad_long_batch_dev(raw.data_ptr() + base, U, B, d_lens.data_ptr(), 0, max_segs, d_atap.data_ptr(), d_n.data_ptr(),
                         d_seg.data_ptr())
    h.sync()
    return d_n.cpu().numpy().view(np.uint32), d_seg.cpu().numpy().view(np.uint32).reshape(B, max(max_segs, 1), 2)[:, :max_segs]


def _both_vad(h, lo, names, acts, max_segs, offs=(0,), U=None):
    pcm, lens = _batch(acts, U)
    B = len(acts)
    want_n, want_seg = lo.vad_long(pcm, plant_atap(B), max_segs, lens)
    v = h.vad_long_batch(pcm, max_segs, 0, lens, atap=plant_atap(B))
    _check(names, v["n_segs"], v["seg_off"], want_n, want_seg, "sr_vad_long_batch")
    for off in offs:
        n, seg = _vad_dev(h, pcm, lens, max_segs, off)
        _check(names, n, seg, want_n, want_seg, "sr_vad_long_batch_dev at offset %d" % off)
    return pcm, lens, want_n


@pytest.mark.gpu
@pytest.mark.parametrize("w", EDGES)
def test_window_edges_bit_exact(handle, w):
    """the edge table with its edge at frame 1 024 w, plus sparse and random strings, through both VAD calls: every
    segment, then cut at MAX_SEGS (the cut cases hold segment MAX_SEGS - 1 or MAX_SEGS open at the edge)"""
    lo = ox.long_oracle()
    cases = edge_cases(w) + (sparse_cases() + random_cases(0x5EED + w, 4) if w == 2 else [])
    names, acts = [c[0] for c in cases], [c[1] for c in cases]
    _, _, n = _both_vad(handle, lo, names, acts, 512, offs=(0, 2))
    assert n.max() <= 512 and (n == 0).sum() == 0
    cut = [b for b, nm in enumerate(names) if nm.startswith("cut")]
    assert len(cut) == 4 and all(MAX_SEGS <= n[b] <= MAX_SEGS + 2 for b in cut)
    _both_vad(handle, lo, names, acts, MAX_SEGS)


@pytest.mark.gpu
def test_window_edges_recognised(handle):
    """sr_recognise_long_batch on the edge table at window 1 against a small bank: every record equals the oracle's"""
    from test_long import _cmp_recognise
    lo, port = ox.long_oracle(), ob.port()
    cases = edge_cases(1)
    pcm, lens = _batch([a for _, a in cases])
    bank, T = ox.synth_bank(4)
    handle.set_bank(bank, T, 4096)
    B = len(cases)
    got = handle.recognise_long_batch(pcm, 128, 0, lens, atap=plant_atap(B))
    want = ox.recognise_long(lo, port, pcm, 0, bank, T, 4096, 128, lens, atap=plant_atap(B))
    _cmp_recognise(got, want)
    assert want["n_segs"].max() <= 128 and (want["segs"]["status"] == 0).sum() > B


# ---- GPU: work splitting -------------------------------------------------------------------------------------------------------
def cpr(U):
    """K11b's chunks (work items of 32 blocks) per recording: its blocks never exceed U / 80 + 1"""
    return (U // 80 + 1 + 31) // 32


def block_grid(U, B, sms):
    """long_block_grid: CTAs of 8 warps, at most two per SM"""
    items, cap = B * cpr(U), 2 * sms
    need = -(-items // 8)
    return (need if need else 1) if need < cap else cap


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _random_acts(rng, B, nfr):
    return [np.asarray(_runs(rng, nfr, 1, 12), np.uint8) for _ in range(B)]


@pytest.mark.gpu
@pytest.mark.parametrize("U", [2559, 7679])
def test_block_pass_grid_strides(handle, U):
    """B * cpr items at n W - 1, n W and n W + 1 (the nearest multiples of cpr) for n = 1, 2, W the grid's warps"""
    lo = ox.long_oracle()
    c = cpr(U)
    assert c == (1 if U == 2559 else 3)
    W = 8 * block_grid(U, 1 << 20, _sms())
    assert W == 16 * _sms()
    rng = np.random.default_rng(U)
    nfr = frames_of(U)
    acts = _random_acts(rng, -(-(2 * W + 1) // c), nfr)
    pcm_all = np.stack([plant(a, U) for a in acts])
    for n in (1, 2):
        for B in sorted({(n * W - 1) // c, -(-n * W // c), -(-(n * W + 1) // c)}):
            assert block_grid(U, B, _sms()) * 8 == W or B * c < W
            pcm = pcm_all[:B]
            want_n, want_seg = lo.vad_long(pcm, plant_atap(B), 4)
            v = handle.vad_long_batch(pcm, 4, 0, atap=plant_atap(B))
            _check(range(B), v["n_segs"], v["seg_off"], want_n, want_seg, "U %d B %d" % (U, B))
            assert want_n.sum() > B // 2


def _last_item_cases(rng, cnb, m):
    """recordings whose last work item holds cnb blocks: nfr = 32 m + cnb - 1 frames. Each ends so that its last frame
    decides a segment: 8 active frames opening at the last frame from the closed state, or 11 inactive ones closing
    there"""
    nfr = 32 * m + cnb - 1
    out = []
    for kind in range(3):
        act = np.asarray(_runs(rng, nfr, 1, 12), np.uint8)
        if kind == 0 and nfr >= 29:
            act[-29:] = [0] * 21 + [1] * 8                  # closed, then an opening whose 8th frame is the last
        elif kind == 1 and nfr >= 20:
            act[-20:] = [1] * 9 + [0] * 11
        out.append(act)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("U", [80 * 101 + 161, 80 * 101 + 162], ids=["odd_U", "even_U"])
def test_short_last_items(U):
    """last items of 1-5 blocks, recordings at every staging parity (odd U: rows alternate; host PCM and _dev PCM at
    offset 0 stage at the row's parity, at offset 2 bytes through plain loads), on a handle whose block workspace holds
    an earlier, quiet call's summaries: a block the kernel skips keeps them and moves a segment"""
    lo = ox.long_oracle()
    rng = np.random.default_rng(U)
    acts, names = [], []
    for cnb in range(1, 6):
        for m in (0, 1, 3):
            if 32 * m + cnb - 1 >= 1 and 80 * (32 * m + cnb - 1) + 160 <= U:
                for k, a in enumerate(_last_item_cases(rng, cnb, m)):
                    for row in ("even", "odd"):                     # rows 2i, 2i + 1: both parities when U is odd
                        acts.append(a)
                        names.append("cnb %d m %d kind %d, %s row" % (cnb, m, k, row))
    assert len({frames_of(80 * len(a) + 160) % 32 for a in acts}) == 5
    h = sr_b200.Handle(0)
    try:
        quiet = np.full((64, 2 * U), 2048, np.uint16)
        h.vad_long_batch(quiet, 4, 0, atap=plant_atap(64))
        pcm, _, _ = _both_vad(h, lo, names, acts, 8, offs=(0, 2), U=U)
        assert pcm.shape[1] == U
    finally:
        h.close()


@pytest.mark.gpu
def test_empty_items_are_skipped_over_several_strides(handle):
    """ragged lens: most items of the batch lie past their recording's end, so next_item skips several strides of them"""
    lo = ox.long_oracle()
    U = 1 << 20
    c, W = cpr(U), 16 * _sms()
    rng = np.random.default_rng(0xE1)
    lens = np.array([0, 161, 500, 0, 0, 240, 2559, 0, 0, 0, 0, 0, 0, 100000, 0, 0, 0, 0, 0, 0, U, U - 1, 999999, U], np.uint32)
    B = len(lens)
    assert B * c > 4 * W and 13 * c > 2 * W                   # the rows before row 13 hold more than two strides of items
    pcm = np.empty((B, U), np.uint16)
    for b in range(B):
        n = int(lens[b])
        pcm[b, :n] = plant(_runs(rng, frames_of(n), 1, 14), n) if n else []
        pcm[b, n:] = np.where(np.arange(U - n) % 2, 4095, 0)
    want_n, want_seg = lo.vad_long(pcm, plant_atap(B), 512, lens)
    v = handle.vad_long_batch(pcm, 512, 0, lens, atap=plant_atap(B))
    _check(range(B), v["n_segs"], v["seg_off"], want_n, want_seg, "empty items")
    n, seg = _vad_dev(handle, pcm, lens, 512)
    _check(range(B), n, seg, want_n, want_seg, "empty items, _dev")
    assert want_n[-4:].min() > 100


@pytest.mark.gpu
@pytest.mark.parametrize("B", [7, 8, 9, 1023, 1024, 1025, 2049])
def test_batch_sizes_recognised(handle, B):
    """recognition past 8 recordings per segment-kernel CTA and 1 024 per prefix-sum pass, max_segs = 2 cutting some rows
    and not others: every record equals the oracle's"""
    from test_long import _cmp_recognise
    lo, port = ox.long_oracle(), ob.port()
    rng = np.random.default_rng(B)
    acts = [np.asarray(_runs(rng, int(rng.integers(1, 200)), 1, 13), np.uint8) for _ in range(B)]
    pcm, lens = _batch(acts)
    bank, T = ox.synth_bank(4)
    handle.set_bank(bank, T, 4096)
    got = handle.recognise_long_batch(pcm, 2, 0, lens, atap=plant_atap(B))
    want = ox.recognise_long(lo, port, pcm, 0, bank, T, 4096, 2, lens, atap=plant_atap(B))
    _cmp_recognise(got, want)
    n = want["n_segs"]
    if B > 100:
        assert (n > 2).sum() > B // 10 and ((n >= 1) & (n <= 2)).sum() > B // 10
        assert (want["segs"]["status"][B - 20:] == 0).sum() > 2
