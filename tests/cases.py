"""Input builders the tests share (TEST INFRASTRUCTURE, CPU only): feature structs and rows, bank slots and planted
banks, random grammars, planted long-form PCM and the digit recordings' banks. Every builder keeps the seeds and the
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
