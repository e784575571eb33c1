"""Input builders the tests share (TEST INFRASTRUCTURE, CPU only): feature structs and rows, bank slots and planted
banks, random grammars, planted long-form PCM, VAD inputs on which every frame of a region decides the segments, noise
windows that give a planned atap, and the digit recordings' banks. Every builder keeps the seeds and the
order of its RNG calls, so a case builds the same bytes wherever it is used. Bare asserts here are not rewritten by
pytest, so each one carries a message."""
import numpy as np

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from refs import MAX_A, MAX_B, MAX_FRM, NULL, slot_rows

DIGITS = ("digits_1_10_a", "digits_1_10_b", "digits_1_9_units_a", "digits_1_9_units_b")


# ---- feature structs and rows ----------------------------------------------------------------------------------------
def make_ftr(rows_list, frm=None):
    """v_ftr_tag structs holding the given [n,12] row arrays; frm: the frm_num of each (default: its row count)"""
    f = np.zeros(len(rows_list), ob.FTR_DTYPE)
    for k, rows in enumerate(rows_list):
        f["frm_num"][k] = len(rows) if frm is None else frm[k]
        f["mfcc_dat"][k][:rows.size] = rows.reshape(-1)
    return f


def band_rows(rng, n, kind):
    """rows of the band DP's cases: "small" in the range of real MFCC rows, "full" +-32 767, "equal" one repeated row"""
    if kind == "small":                      # the range of real MFCC rows
        return rng.integers(-3000, 3001, (n, 12)).astype(np.int16)
    if kind == "full":                       # +-32767: d ~ 65 500 on all but 1 in 4096 cells
        return (rng.choice([-1, 1], (n, 12)) * 32767).astype(np.int16)
    if kind == "equal":                      # d = 0 everywhere: every min of the recurrence is a tie
        return np.tile(np.array([7, -3, 11, 0, -25, 4, 9, -1, 2, 3, -8, 6], np.int16), (n, 1))
    raise ValueError(kind)


def tie_rows(rng, n, kind):
    """rows of the symmetric and any-rate matchers' cases: "tie" from {0, 1}, "full" +-32 767, otherwise -400 .. 399"""
    if kind == "tie":
        return rng.integers(0, 2, (n, 12)).astype(np.int16)
    if kind == "full":
        return rng.choice(np.array([-32767, 32767], np.int16), (n, 12))
    return rng.integers(-400, 400, (n, 12)).astype(np.int16)


def guard_edge_shapes():
    """every (I, M) on the edges of the 2:1 guard (M = 2I, I = 2M and one either side, both inside 1..119) and the corners"""
    s = {(1, 1), (1, 2), (2, 1), (119, 119), (60, 119), (119, 60)}
    for a in range(1, MAX_FRM + 1):
        for b in (2 * a - 1, 2 * a, 2 * a + 1):
            if 1 <= b <= MAX_FRM:
                s |= {(a, b), (b, a)}
    return sorted(s)


def band_cases():
    """(name, utterances, templates): utterance k and template k have k + 1 rows, so each case holds every (I, M) with
    I, M in 1..119 (the guard edges among them) and 119 templates (three full 32-wide tiles and a remainder tile)"""
    rng = np.random.default_rng(0xBA4D)
    lens = range(1, MAX_FRM + 1)
    small_u = [band_rows(rng, n, "small") for n in lens]
    full_u = [band_rows(rng, n, "full") for n in lens]
    full_t = [band_rows(rng, n, "full") for n in lens]
    for k in (59, 118):                      # 60 and 119 rows: the largest local distance on every cell
        full_u[k], full_t[k] = np.tile(MAX_A, (k + 1, 1)), np.tile(MAX_B, (k + 1, 1))
    return [("small", small_u, [band_rows(rng, n, "small") for n in lens]),
            ("full", full_u, full_t),
            ("equal", [band_rows(rng, n, "equal") for n in lens], [band_rows(rng, n, "equal") for n in lens]),
            ("self", small_u, [x.copy() for x in small_u])]


def inputs(rng, frms):
    """feature structs of frms[k] frames (1..119 rows of tie_rows; frm_num 0 and 120 keep 1 and 119 rows)"""
    return make_ftr([tie_rows(rng, max(f, 1) if f <= 119 else 119, ("small", "tie", "full")[k % 3])
                     for k, f in enumerate(frms)], frm=frms)


def bank_planted(rng, T):
    """T template slots of 1..119 rows, with an erased slot, an unsigned slot, frm_num 0 and frm_num 120 planted"""
    frms = rng.integers(1, 120, T)
    f = inputs(rng, frms)
    valid = np.ones(T, bool)
    bank = sr_b200.make_bank(f, 4096)
    if T >= 4:
        bank[T // 4] = 0xFF                                  # erased flash
        valid[T // 3] = False
        bank[T // 3, 0:2] = 0x00                             # unsigned (save_sign 0)
        bank[T // 2, 2:4] = 0                                # frm_num 0
        bank[T - 1, 2:4] = (120, 0)                          # frm_num 120
    return bank


# ---- bank slots ------------------------------------------------------------------------------------------------------
def make_slot(rows, stride, sign=sr_b200.SAVE_MASK, frm=None):
    """one bank slot of stride bytes holding rows (0xFF past them); frm: its frm_num (default: the row count)"""
    s = np.full(stride, 0xFF, np.uint8)
    n = len(rows) if frm is None else frm
    s[:4] = np.frombuffer(np.array([sign, n], np.uint16).tobytes(), np.uint8)
    s[4:4 + rows.size * 2] = np.frombuffer(np.ascontiguousarray(rows, np.int16).tobytes(), np.uint8)
    return s


def random_groups(rng, G, K, stride, fmin=3, fmax=24, plant=True):
    """G groups of K slots of random features (lengths fmin..fmax, some repetitions of one word plus noise); with plant,
    the invalid cases go into the first groups: an erased slot, frm_num 0, frm_num 120, an unsigned slot, a member the
    2:1 guard rejects against the others, and an all-empty group"""
    bank = np.full((G * K, stride), 0xFF, np.uint8)
    for g in range(G):
        n0 = int(rng.integers(fmin, fmax + 1))
        base = rng.integers(-3000, 3001, (n0, 12))
        for k in range(K):
            n = int(np.clip(n0 + rng.integers(-n0 // 3, n0 // 3 + 1), 1, MAX_FRM))
            idx = np.minimum((np.arange(n) * n0) // n, n0 - 1)
            rows = base[idx] + rng.integers(-400, 401, (n, 12))
            bank[g * K + k] = make_slot(rows, stride)
    if plant and G >= 3:
        k_last = K - 1
        if K >= 2:
            bank[0 * K + k_last] = 0xFF                                           # erased
            bank[1 * K + k_last] = make_slot(np.zeros((0, 12)), stride, frm=0)    # frm_num 0
        if K >= 3:
            bank[0 * K + 1] = make_slot(rng.integers(-9, 9, (5, 12)), stride, frm=120)   # frm_num 120
            bank[1 * K + 1] = make_slot(rng.integers(-3000, 3001, (10, 12)), stride, sign=0)   # unsigned
            n = slot_rows(bank[2 * K])[1]
            bank[2 * K + 1] = make_slot(rng.integers(-3000, 3001, (min(2 * n + 3, MAX_FRM), 12)), stride)   # guard rejects
        bank[(G - 1) * K:G * K] = 0xFF                                            # all empty
    return bank


def word_bank(T, seed, erase=(), dup=(), trunc=None):
    """T slots of 4 096 bytes from synthetic one-word templates: command c's four slots are one word with one row dropped each (row
    k * 7, none for k = 0), optionally cut to trunc(t) frames; dup (a, b) copies slot a into slot b; erase: unsigned"""
    n_cmd = (T + 3) // 4
    e = ob.recognise_pinned(ob.best_oracle(), sr_b200.synth_pcm_host(n_cmd, 8000, seed), 2400, None, 0, 4096)
    ftr = np.zeros(4 * n_cmd, ob.FTR_DTYPE)
    for t in range(4 * n_cmd):
        f = e["ftr"][t // 4]
        n = int(f["frm_num"])
        rows = f["mfcc_dat"][:n * 12].reshape(n, 12)
        x = rows if t % 4 == 0 else np.delete(rows, min((t % 4) * 7, n - 1), axis=0)
        if trunc:
            x = x[:trunc(t)]
        ftr[t]["frm_num"] = len(x)
        ftr[t]["mfcc_dat"][:x.size] = x.reshape(-1)
    for a, b in dup:
        ftr[b] = ftr[a]
    valid = np.ones(T, bool)
    valid[list(erase)] = False
    return sr_b200.make_bank(ftr[:T], 4096, valid)


def headroom_bank(seed):
    """8 slots of word_bank(8, seed) (slot 6 unsigned, slot 3 a copy of slot 0) with +32 767 and -32 767 in
    coefficients 0 and 1 of every row, and command 1's rows +32 767 in coefficient 2 as well: every greedy and symmetric
    score of a synthetic utterance is above 32 768 (a margin rule's q d1 passes 2^31 at q = 65 535), and command 1, the
    runner-up, scores about a quarter more than command 0"""
    T = 8
    f = np.ascontiguousarray(word_bank(T, seed)[:, :ob.FTR_DTYPE.itemsize]).view(ob.FTR_DTYPE).reshape(T).copy()
    f[3] = f[0]
    rows = f["mfcc_dat"].reshape(T, MAX_FRM, 12)
    rows[:, :, 0], rows[:, :, 1] = 32767, -32767
    rows[4:, :, 2] = 32767
    valid = np.ones(T, bool)
    valid[6] = False
    return sr_b200.make_bank(f, 4096, valid)


# ---- connected words and grammars ------------------------------------------------------------------------------------
def draw(rng, n, kind):
    """n feature rows: "tie" from {0, 1}, "full" +-32 767, "equal" one repeated row, otherwise -3000 .. 3000"""
    if kind == "tie":                                     # rows from {0, 1}: ties everywhere
        return rng.integers(0, 2, (n, 12)).astype(np.int16)
    if kind == "full":                                    # +-32767
        return (rng.choice([-1, 1], (n, 12)) * 32767).astype(np.int16)
    if kind == "equal":
        return np.tile(np.array([7, -3, 11, 0, -25, 4, 9, -1, 2, 3, -8, 6], np.int16), (n, 1))
    return rng.integers(-3000, 3001, (n, 12)).astype(np.int16)


def random_bank(rng, T, kind, stride=2880, fmin=1, fmax=8, plant=True):
    """T slots of fmin..fmax frames; with plant, non-members mixed in: erased, unsigned, frm_num 0 and frm_num 120"""
    bank = np.stack([make_slot(draw(rng, int(rng.integers(fmin, fmax + 1)), kind), stride) for _ in range(T)]) if T else \
        np.zeros((0, stride), np.uint8)
    if plant and T >= 3:
        for t in rng.choice(T, min(T - 1, max(1, T // 4)), replace=False):
            c = int(rng.integers(4))
            bank[t] = (np.full(stride, 0xFF, np.uint8) if c == 0 else make_slot(draw(rng, 3, kind), stride, sign=0)
                       if c == 1 else make_slot(np.zeros((0, 12)), stride, frm=0) if c == 2
                       else make_slot(draw(rng, 5, kind), stride, frm=120))
    return bank


def random_grammar(rng, S=None):
    """an NFA of 1-5 states: overlapping arcs (shared endpoints, overlapping command masks), unreachable or dead states,
    a random final mask"""
    S = int(rng.integers(1, 6)) if S is None else S
    arcs = []
    for _ in range(int(rng.integers(1, 2 * S + 2))):
        a, b = int(rng.integers(S)), int(rng.integers(S))
        m = int(rng.integers(1, 4)) if rng.random() < 0.6 else int(rng.integers(0, 2 ** 32))
        arcs.append((a, b, m))
    F = int(rng.integers(1, 2 ** S))
    return (S, F, arcs)


def partition_grammar(rng, S, n_cmd=32):
    """S states; every command is assigned to one state, whose incoming arcs (from state 0, from itself and from a random
    state) carry exactly its commands: the copies are the bank's members, once each"""
    own = rng.integers(0, S, n_cmd)
    arcs = []
    for s in range(S):
        m = int(sum(1 << c for c in range(n_cmd) if own[c] == s))
        if m:
            arcs += [(0, s, m), (s, s, m), (int(rng.integers(S)), s, m)]
    return (S, int(rng.integers(1, 2 ** S)) | 1 << (S - 1), arcs)


# ---- long recordings -------------------------------------------------------------------------------------------------
def frames_of(n):
    """frames i = 80k while i < n - 160 (VAD.C:121)"""
    return -(-(n - 160) // 80) if n > 160 else 0


PLANT_ATAP = (2048, 100, 0, 0xFFFFFFFF)     # mid, n_thl, z_thl, s_thl: a frame is active on one band crossing


def plant(act, n=None):
    """PCM of n samples (default 80 N + 160) whose N = len(act) frames are active exactly where act is 1 under PLANT_ATAP:
    every sample is in band except one priming sample at position 0 and one sample at 80(k+1) per active frame k,
    alternately above and below the band"""
    act = np.asarray(act, np.uint8)
    n = 80 * len(act) + 160 if n is None else n
    assert frames_of(n) == len(act), (n, len(act))
    pcm = np.full(n, 2048, np.uint16)
    pcm[0] = 1947                                           # below the band: last_sig = 1 before frame 0
    k = np.flatnonzero(act)
    pcm[80 * (k + 1)] = np.where(np.arange(len(k)) % 2 == 0, 2148, 1947)
    return pcm


def plant_atap(B):
    a = np.zeros(B, ob.ATAP_DTYPE)
    a["mid_val"], a["n_thl"], a["z_thl"], a["s_thl"] = PLANT_ATAP
    return a


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


def synth_long_poisoned(lengths, U, seed):
    """recordings of the given lengths (many words each) in rows of U samples, poisoned past their length"""
    pcm = ox.synth_long(len(lengths), U, seed)
    for b, n in enumerate(lengths):
        pcm[b, n:] = np.where(np.arange(U - n) % 2, 4095, 0)
    return pcm


# ---- banks of templates ----------------------------------------------------------------------------------------------
def bank_of_ftr(ftr_, valid_slots=None):
    """one template per feature struct, template k in slot 4k (cmd = k); the other slots erased"""
    K = len(ftr_)
    ftr4 = np.zeros(4 * K, ob.FTR_DTYPE)
    ftr4[0::4] = ftr_
    valid = np.zeros(4 * K, bool)
    valid[0::4] = True
    return sr_b200.make_bank(ftr4, 4096, valid), 4 * K


def real_speech_pairs():
    """(enrolled recording, recognised twin) of the four digit recordings"""
    return ((DIGITS[0], DIGITS[1]), (DIGITS[1], DIGITS[0]), (DIGITS[2], DIGITS[3]), (DIGITS[3], DIGITS[2]))


def digit_bank(port, lo, a):
    """template k = segment k of recording a, in slot 4k (the other slots unsigned)"""
    ea = ox.recognise_long(lo, port, a[None], 2400, None, 0, 4096, 32)
    ma = int(ea["n_segs"][0])
    f = ox.ftr_of_segments(port, a[None], ea["atap"], [(0, int(s["start"]), int(s["end"]) if s["end"] != NULL
                                                        else int(s["start"])) for s in ea["segs"][0, :ma]])
    ftr4 = np.zeros(4 * ma, ob.FTR_DTYPE)
    ftr4[0::4] = f
    valid = np.zeros(4 * ma, bool)
    valid[0::4] = True
    return sr_b200.make_bank(ftr4, 4096, valid), 4 * ma, ma


# ---- VAD inputs on which every frame of a region decides the segments ------------------------------------------------
# Frame k of VAD.C:121-164 reads blocks k and k + 1 (80 samples each). The builder fills the blocks in order: once block k
# is placed, frame k's features depend only on block k + 1, which is drawn until frame k lands exactly on its target. In
# the critical region the targets sit on the thresholds (an active frame one unit above, an inactive frame exactly at it)
# and the activity is runs of exactly 8 active and 11 inactive frames, so a +-1 error in any critical frame's frm_sum or
# frm_zero flips its activity, and every flip changes the segments.
U32 = 0xFFFFFFFF


def vad_atap(mid, n_thl, z_thl, s_thl):
    a = np.zeros(1, sr_b200.ATAP_DTYPE)
    a["mid_val"], a["n_thl"], a["z_thl"], a["s_thl"] = mid, n_thl, z_thl, s_thl
    return a


class Bands:
    """the band of an atap (VAD.C:112-113, u32): value ranges [lo, hi] of the classes 0 (in band), 1 (below b_thl) and
    2 (at or above a_thl) among u16 samples, None where a class has no value"""

    def __init__(self, atap):
        a0 = atap.reshape(-1)[0]
        self.mid, self.n_thl = int(a0["mid_val"]), int(a0["n_thl"])
        self.z_thl, self.s_thl = int(a0["z_thl"]), int(a0["s_thl"])
        self.a, self.b = (self.mid + self.n_thl) & U32, (self.mid - self.n_thl) & U32
        top = min(self.a, 65536)
        self.rng = {2: (self.a, 65535) if self.a <= 65535 else None,
                    1: (0, min(self.b, top) - 1) if min(self.b, top) > 0 else None,
                    0: (self.b, top - 1) if self.b < top else None}
        self.edge = {2: [self.a], 1: [min(self.b, top) - 1], 0: [self.b, top - 1]}   # values on a class boundary

    def dev(self, c):
        lo, hi = self.rng[c]
        m = self.mid
        return (0, max(m - lo, hi - m)) if lo <= m <= hi else ((lo - m, hi - m) if m < lo else (m - hi, m - lo))

    def value(self, c, d, rng):
        lo, hi = self.rng[c]
        v = [x for x in (self.mid + d, self.mid - d) if lo <= x <= hi]
        return v[int(rng.integers(len(v)))]

    def cls(self, x):
        x = np.asarray(x, np.int64)
        return np.where(x >= self.a, 2, np.where(x < self.b, 1, 0)).astype(np.int8)


def scan_zero(cls, lo, hi, last):
    """VAD.C:132-157 over samples lo .. hi: alternations counted at positions lo + 1 .. hi with last_sig entering at lo;
    (count, last_sig after sample hi - 1)"""
    cnt = 0
    for p in range(lo, hi):
        if cls[p]:
            last = int(cls[p])
        w = cls[p + 1]
        if w and last and w != last:
            cnt += 1
    return cnt, last


def _block(rng, bd, c_prev, r, B, quiet, bare=False):
    """80 samples whose markers make exactly r alternations after last_sig c_prev (None: any) and whose |x - mid| sum to
    B (None: any); bare: no marker before position 79, so the frame that starts here carries its class in from an
    earlier block. None when the draw fails"""
    classes = [c for c in (1, 2) if bd.rng[c] is not None]
    if bare:
        if bd.rng[0] is None or (r or 0) > (1 if c_prev else 0):
            return None
        m = int(r or 0)
    elif bd.rng[0] is None:
        m = 80
    elif r is None:
        m = 0 if quiet or rng.random() < 0.4 else int(rng.integers(1, 8))
    else:
        m = r + (1 if (c_prev == 0 and r) else 0)
        m = 0 if (r == 0 and rng.random() < 0.4) else min(80, m + int(rng.integers(0, 4)))
    if r and len(classes) < 2:
        return None
    slots = ([0] if c_prev else []) + list(range(1, m))
    k = r if r is not None else (int(rng.integers(0, len(slots) + 1)) if len(classes) == 2 else 0)
    if k > len(slots):
        return None
    flip = set(rng.choice(slots, k, replace=False).tolist()) if k else set()
    cur = c_prev if c_prev in classes else classes[int(rng.integers(len(classes)))]
    seq = []
    for i in range(m):
        if i in flip:
            cur = 3 - cur
        seq.append(cur)
    pos = [79] if bare and m else sorted(rng.choice(80, m, replace=False).tolist()) if m < 80 else list(range(80))
    if 0 < m < 80 and not bare:
        for want in (0, 1, 78, 79):
            if want not in pos and rng.random() < 0.25:
                pos[int(rng.integers(m))] = want
        pos = sorted(set(pos))
        if len(pos) != m:
            return None
    cl = np.zeros(80, np.int8)
    cl[pos] = seq
    if bd.rng[0] is None and (cl == 0).any():
        return None
    lo = np.array([bd.dev(int(c))[0] for c in cl], np.int64)
    hi = np.array([bd.dev(int(c))[1] for c in cl], np.int64)
    x = np.zeros(80, np.int64)
    pin = np.zeros(80, bool)
    for i in range(80):                                   # boundary values: a_thl, b_thl - 1, b_thl, a_thl - 1
        if rng.random() < (0.3 if cl[i] else 0.15):
            v = bd.edge[int(cl[i])][int(rng.integers(len(bd.edge[int(cl[i])])))]
            if 0 <= v <= 65535 and bd.cls([v])[0] == cl[i] and (cl[i] or B is None or abs(v - bd.mid) <= B // 16):
                x[i], pin[i] = v, True
    spread = np.minimum(hi - lo, 40 if quiet else 400)
    d = lo + (rng.random(80) * (spread + 1)).astype(np.int64)
    d[pin] = np.abs(x[pin] - bd.mid)
    if B is not None:
        diff = B - int(d.sum())
        free = [i for i in rng.permutation(80).tolist() if not pin[i]]
        for t in range(2):
            for j, i in enumerate(free):
                if diff == 0:
                    break
                room = hi[i] - d[i] if diff > 0 else d[i] - lo[i]
                share = abs(diff) if t else -(-abs(diff) // (len(free) - j))
                step = min(room, share)
                d[i] += step if diff > 0 else -step
                diff += -step if diff > 0 else step
        if diff:
            return None
    for i in range(80):
        if not pin[i]:
            x[i] = bd.value(int(cl[i]), int(d[i]), rng)
    return x.astype(np.uint16)


def critical_targets(nfr, groups, family, bd):
    """per frame: active, critical, and the (lo, hi) each feature must land in. groups: the first frames of runs of 8
    active frames, each followed by 11 inactive ones; the critical region of a group is the frame before it through the
    11th inactive frame"""
    act, crit = np.zeros(nfr, bool), np.zeros(nfr, bool)
    for g in groups:
        assert g >= 1 and g + 19 <= nfr, (g, nfr)
        act[g:g + 8] = True
        crit[g - 1:g + 19] = True
    z, s = bd.z_thl, bd.s_thl
    zt, st = [], []
    for k in range(nfr):
        a = int(act[k])
        if not crit[k]:
            zt.append((0, z)), st.append((0, s))
        elif family == "sum":                              # frm_sum decides, frm_zero never can (z_thl >= 159)
            zt.append((0, z)), st.append((s + a, s + a))
        elif family == "zero":                             # frm_zero decides, frm_sum stays at or under s_thl
            zt.append((z + a, z + a)), st.append((0, s))
        elif family == "mixz":                             # frm_zero decides, frm_sum exactly at s_thl
            zt.append((z + a, z + a)), st.append((s, s))
        else:                                              # "mixs": frm_sum decides, frm_zero exactly at z_thl
            assert family == "mixs", family
            zt.append((z, z)), st.append((s + a, s + a))
    return act, crit, zt, st


def critical_pcm(rng, atap, family, nfr, groups, n=None, prefix=None, bsum=(0.3, 0.7), bare=()):
    """PCM of n samples (default 80 nfr + 160) with nfr frames, critical around each of `groups` (critical_targets);
    prefix: samples the PCM starts with (a multiple of 80, e.g. a noise window; its frames must be inactive); bsum: the
    share of s_thl a block's sum is kept in where a frame's sum is pinned; bare: blocks with no marker before position 79
    (frame k then enters with a class from before block k). Returns (pcm, act, crit)."""
    bare = set(bare)
    bd = Bands(atap)
    n = 80 * nfr + 160 if n is None else n
    assert frames_of(n) == nfr and n >= 80 * nfr + 80, (n, nfr)
    act, crit, zt, st = critical_targets(nfr, groups, family, bd)
    x = np.zeros(80 * (nfr + 1), np.int64)
    cls = np.zeros(80 * (nfr + 1), np.int8)
    dev = np.zeros(nfr + 1, np.int64)                     # per-block sum of |x - mid|
    zfree, sfree = bd.z_thl >= 159, bd.s_thl >= 80 * 160 * 65535 // 2
    p0 = 0
    if prefix is not None:
        assert len(prefix) % 80 == 0 and len(prefix) <= len(x), len(prefix)
        x[:len(prefix)] = prefix
        cls[:len(prefix)] = bd.cls(prefix)
        dev[:len(prefix) // 80] = np.abs(np.asarray(prefix, np.int64) - bd.mid).reshape(-1, 80).sum(1)
        p0 = len(prefix) // 80
    init = [0] * (nfr + 1)                                 # last_sig entering frame k
    last = 0
    for k in range(nfr):
        # last_sig entering frame k: class of the last marker at or before sample 80k + 78 (the first frame: none)
        init[k] = last if k else 0
        if k + 1 < p0:
            _, last = scan_zero(cls, 80 * k, 80 * k + 159, init[k])
            continue
        if k == 0 and p0 == 0:                             # block 0: quiet, markers of one class at most
            b, s0 = None, st[0][0]
            lo_b, hi_b = (s0 - int(bsum[1] * bd.s_thl), s0 - int(bsum[0] * bd.s_thl)) if s0 == st[0][1] else (0, s0 // 8)
            r0 = 0 if zfree or not crit[0] else int(rng.integers(0, min(2, zt[0][0]) + 1))   # frame 0's own alternations
            while b is None:
                b = _block(rng, bd, 0, None if zfree else r0, None if sfree else int(rng.integers(lo_b, hi_b + 1)), True)
            x[:80], cls[:80], dev[0] = b, bd.cls(b), int(np.abs(b.astype(np.int64) - bd.mid).sum())
        own, _ = scan_zero(cls, 80 * k, 80 * k + 79, init[k])
        c_prev = int(cls[80 * k + 79]) or scan_zero(cls, 80 * k, 80 * k + 79, init[k])[1]
        for attempt in range(400):
            zlo, zhi = zt[k]
            slo, shi = st[k]
            quiet = not crit[k]
            if zfree:
                r = None
            elif zlo == zhi:
                r = zlo - own
            else:                                          # an inactive frame off the region: few alternations
                lo_r = max(0, zlo - own)
                r = lo_r if rng.random() < 0.7 else int(rng.integers(lo_r, max(lo_r, zhi - own) + 1))
            if sfree:
                B = None
            elif slo == shi:
                B = slo - int(dev[k])
            else:
                top = shi - int(dev[k])
                lo_b, hi_b = 0, top // 4 if quiet else top
                if k + 1 < nfr and st[k + 1][0] == st[k + 1][1]:     # the next frame's sum is pinned: leave it room
                    lo_b = max(0, st[k + 1][0] - int(bsum[1] * bd.s_thl))
                    hi_b = min(top, st[k + 1][0] - int(bsum[0] * bd.s_thl))
                B = int(rng.integers(lo_b, hi_b + 1)) if 0 <= lo_b <= hi_b else -1
            if r is not None and r < 0 or B is not None and B < 0:
                raise AssertionError("frame %d: no block %d can reach the target" % (k, k + 1))
            b = _block(rng, bd, c_prev, r, B, quiet, k + 1 in bare and attempt < 200)   # bare where it can be
            if b is None:
                continue
            bc = bd.cls(b)
            o = 80 * (k + 1)
            cls[o:o + 80] = bc
            x[o:o + 80] = b
            dev[k + 1] = int(np.abs(b.astype(np.int64) - bd.mid).sum())
            zk, last_k = scan_zero(cls, 80 * k, 80 * k + 159, init[k])
            sk = int(dev[k] + dev[k + 1])
            assert zt[k][0] <= zk <= zt[k][1] and st[k][0] <= sk <= st[k][1], (k, zk, sk, zt[k], st[k])
            if k + 1 < nfr:                                # frame k + 1 must stay reachable by block k + 2
                own1, _ = scan_zero(cls, o, o + 79, last_k)
                zlo1, zhi1 = zt[k + 1]
                need = zlo1 - own1
                if not zfree and (own1 > zhi1 or need > max(2, bd.z_thl) + 2 or (k + 2 in bare and attempt < 200 and need > 1)):
                    continue
                slo1, shi1 = st[k + 1]
                if not sfree and slo1 == shi1 and not (bsum[0] * bd.s_thl <= slo1 - dev[k + 1] <= bsum[1] * bd.s_thl):
                    continue
                if not sfree and dev[k + 1] > shi1:
                    continue
            last = last_k
            break
        else:
            raise AssertionError("frame %d: no block %d found" % (k, k + 1))
    pcm = np.zeros(n, np.uint16)
    pcm[:len(x)] = x
    if n > len(x):                                         # samples no frame reads
        pcm[len(x):] = rng.integers(0, 65536, n - len(x))
    return pcm, act, crit


def noise_window(mid, n_thl, s_thl, n_len=2400):
    """n_len samples on which noise_atap (VAD.C:22-71) gives exactly mid_val = mid, n_thl and s_thl (z_thl is always 2):
    every sample in band (the largest deviation of each 240-sample block is one sample at mid - n_thl = b_thl, which is
    not below the band), deviations spread evenly so that no frame over the window is active"""
    nf = n_len // 160
    A = next(a for a in range(s_thl * 10 // 11 - 2, s_thl * 10 // 11 + 3) if a * 11 // 10 == s_thl)
    T = A * nf                                            # sum of |x - mid|: abs_sum / nf = A, s_thl = A * 11 / 10
    N = T // 2
    P = T - N                                             # sum stays in [mid n_len, mid n_len + n_len): mean = mid
    pins = n_len // 240
    d = np.zeros(n_len, np.int64)
    pos, neg = np.arange(0, n_len, 2), np.arange(1, n_len, 2)
    pin = neg[::120][:pins]                               # one per 240-sample block
    rest = np.setdiff1d(neg, pin)
    d[pos] = -(P // len(pos))
    d[pos[:P % len(pos)]] -= 1
    Nr = N - pins * n_thl
    d[rest] = Nr // len(rest)
    d[rest[:Nr % len(rest)]] += 1
    d[pin] = n_thl
    x = mid - d                                           # d > 0: below mid
    assert d[pos].min() > -n_thl and 0 <= d[rest].max() <= n_thl and Nr >= 0 and x.min() >= 0 and x.max() <= 65535, \
        (mid, n_thl, s_thl)
    return x.astype(np.uint16), vad_atap(mid, n_thl, 2, s_thl)


# the coverage table: what the critical frames of a case set must contain between them
COVER_UNITS = ("alternation inside block k", "alternation inside block k+1", "alternation across blocks k, k+1",
               "carried class from block k (positions 0-78)", "marker at block k position 79 not carried",
               "carried class from the previous block", "carried class from many blocks back", "no carried class",
               "no carried class at frame 0", "first marker at position 0", "first marker later",
               "counted marker at block position 0", "counted marker at block position 1",
               "counted marker at block position 78", "counted marker at block position 79",
               "sample at a_thl", "sample at b_thl", "sample at b_thl - 1", "b_thl wrapped",
               "a_thl = 0, sums decide", "a_thl > 0xFFFF, sums decide", "b_thl = 0, sums decide")
COVER_PLACES = ("first frame of a 32-frame pass", "class carried into the first frame of a 32-frame pass", "frame across a 2 560-sample chunk edge", "split8 tail",
                "1 024-frame window edge", "last frame")


def frame_cover(pcm, atap, k, init, nfr, family):
    """the coverage-table entries critical frame k of a capture of nfr frames exercises (init: last_sig entering it)"""
    bd = Bands(atap)
    out = set()
    o = 80 * k
    if family in ("sum", "mixs"):
        if bd.a == 0:
            out.add("a_thl = 0, sums decide")
        if bd.a > 0xFFFF:
            out.add("a_thl > 0xFFFF, sums decide")
        if bd.b == 0 and family == "mixs":
            out.add("b_thl = 0, sums decide")
    if k % 32 == 0 and k:
        out.add("first frame of a 32-frame pass")
    if k % 32 == 31:
        out.add("frame across a 2 560-sample chunk edge")
    r = (nfr + 1) % 32
    if 1 <= r <= 4 and k + 1 >= nfr + 1 - r:
        out.add("split8 tail")
    if k >= 1023 and k % 1024 in (0, 1023):
        out.add("1 024-frame window edge")
    if k == nfr - 1:
        out.add("last frame")
    if family == "sum" or bd.z_thl >= 159:
        return out
    x = np.asarray(pcm[o:o + 160], np.int64)
    cls = bd.cls(x)
    if bd.b > 0xFFFF:
        out.add("b_thl wrapped")
    mk = np.flatnonzero(cls)
    before = bd.cls(np.asarray(pcm[:o + 79], np.int64))
    prior = np.flatnonzero(before)                         # markers at or before sample 80k + 78
    src = None if not len(prior) or k == 0 else prior[-1] - o
    if len(mk):
        F, cF = int(mk[0]), int(cls[mk[0]])
        if F > 0 and init and init != cF:
            out.add("first marker later")
            out.add("carried class from block k (positions 0-78)" if src >= 0 else
                    "carried class from the previous block" if src >= -80 else "carried class from many blocks back")
            if src < 0 and k % 32 == 0:
                out.add("class carried into the first frame of a 32-frame pass")
        if F == 0 and k and init and init != cF:
            out.add("first marker at position 0")
        if k and not init and F > 0:
            out.add("no carried class")
        if k == 0 and F > 0:
            lcA = [int(cls[p]) for p in mk if p <= 78]
            if lcA and lcA[-1] != cF:
                out.add("no carried class at frame 0")
        if k and cls[79] and F > 0:
            c79 = int(cls[79])
            if (init != 0 and init != cF) != (c79 != cF):
                out.add("marker at block k position 79 not carried")
    last = init
    for h in range(159):
        if cls[h]:
            last = int(cls[h])
        p = h + 1
        if x[p] == bd.b and last == 2 and bd.b <= 65535:
            out.add("sample at b_thl")
        if cls[p] and last and cls[p] != last:
            prev = [q for q in mk if q < p]
            if prev:
                q = prev[-1]
                out.add("alternation inside block k" if p < 80 else "alternation inside block k+1" if q >= 80 else
                        "alternation across blocks k, k+1")
                for v in (x[p], x[q]):
                    if v == bd.a:
                        out.add("sample at a_thl")
                    if v == bd.b - 1 and bd.b <= 65535:
                        out.add("sample at b_thl - 1")
            if p % 80 in (0, 1, 78, 79):
                out.add("counted marker at block position %d" % (p % 80))
    return out
