"""A plain stage reference of get_mfcc (MFCC.C:86-191) for one frame at a time (TEST INFRASTRUCTURE, CPU only), in the
reference geometry (160 / 80 / 1024, 512 bins) and in GEOM_B (200 / 80 / 256, 128 bins). Written from MFCC.C's
definitions and sharing no code with oracle/sr_oracle.c: the windowed samples, the spectrum (the oracle's FFT
restatement, pinned on its own to the asm and to the exact DFT), float32 magnitudes, u32 energies, the 24 filter sums
summed bin by bin over each filter's range, log*100 by a search over the committed threshold table, and the truncated
DCT. Every stage is kept, so tests can ask which filter sums a frame's coefficients are sensitive to. The tables of
the reference geometry are the reference's own (tests/golden/ref_tables.npz); GEOM_B's come from tools/gen_tables.py,
which tests/test_tables.py holds to the committed header."""
import functools
import os
import re
import sys

import numpy as np

import oracle_bind as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_tables  # noqa: E402

M32 = np.uint64(0xFFFFFFFF)
L_MAX = 2218                                    # (u32)(log(2^32 - 1) * 100)


def _header_table(name, n):
    text = open(os.path.join(ROOT, "stm32-speech-recognition_b200", "csrc", "sr_tables.h")).read()
    body = re.search(r"\b%s\[%d\] = \{([^}]*)\}" % (name, n), text).group(1)
    return [int(x) for x in body.replace("\n", "").split(",") if x.strip()]


# thr[L] = the least v with (u32)(log(v) * 100) >= L, L = 0 .. 2218 (the committed table without its pad entry)
THR = np.array(_header_table("sr_tab_log_thr", 2220)[:L_MAX + 1], np.uint64)


class Geometry:
    """frame length, hop, FFT size and the tables of one front end; filter h covers bins [lo[h], hi[h]) with the
    weights of its parity (MFCC.C:136-162: even filters tri_even, odd filters tri_odd)"""

    def __init__(self, name, frame, n_fft, hamm, cen, tri_even, tri_odd, dct):
        self.name, self.frame, self.hop, self.n_fft, self.bins = name, frame, 80, n_fft, n_fft // 2
        self.hamm = np.asarray(hamm, np.int64)
        self.cen = [int(c) for c in cen]
        self.w = [np.asarray(tri_even, np.uint64), np.asarray(tri_odd, np.uint64)]
        self.dct = np.asarray(dct, np.int64).reshape(12, 24)
        lo = [0] + [self.cen[h - 1] for h in range(1, 24)]                 # pow_spct[0] starts at bin 0
        hi = [self.cen[h + 1] for h in range(23)] + [self.bins]            # pow_spct[23] ends at fft_point / 2
        self.lo, self.hi = lo, hi

    def frames_of(self, n):
        """frame count of an n-sample segment (MFCC.C:102-107): 0 below one frame and above vv_frm_max = 119"""
        if n < self.frame:
            return 0
        f = (n - self.frame) // self.hop + 1
        return 0 if f > 119 else f


def _ref_geometry():
    z = np.load(os.path.join(ROOT, "tests", "golden", "ref_tables.npz"))
    return Geometry("A", 160, 1024, z["hamm"], z["tri_cen"], z["tri_even"], z["tri_odd"], z["dct_arg"])


def _geom_b():
    cen, odd, even = gen_tables.tri_tables(gen_tables.FRQ_MAX_B)
    return Geometry("B", gen_tables.FRAME_LEN_B, gen_tables.FFT_POINT_B, gen_tables.hamm_table(gen_tables.FRAME_LEN_B),
                    cen, even, odd, gen_tables.dct_table())


GEOM_A, GEOM_B = _ref_geometry(), _geom_b()


def _cdiv(a, d):
    """C division of int64 arrays: truncates toward zero"""
    return np.sign(a) * (np.abs(a) // d)


def windowed(cur, prv, mid, hamm):
    """vc_temp of MFCC.C:118-121: ((x - mid) - (x[-1] - mid) * 95 / 100) * hamm / 1000 in s32 with truncating
    divisions, stored as s16. cur, prv [n, L] samples, mid [n]"""
    mid = np.asarray(mid, np.int64).reshape(-1, 1)
    t = (cur.astype(np.int64) - mid) - _cdiv((prv.astype(np.int64) - mid) * 95, 100)
    return _cdiv(t * hamm[None, :], 1000).astype(np.int16)


def magnitude(spec, bins):
    """fft() of MFCC.C:49-59 on packed (re | im << 16) bins: real * real + imag * imag in s32, then
    (u32)(sqrtf((float)pw) * 10) -- each step an IEEE float32 operation, the product truncated. A negative pw (only
    re = im = -32768) takes sqrtf's NaN, which converts to 0"""
    s = spec[:, :bins]
    re = (s & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.int64)
    im = (s >> 16).astype(np.uint16).view(np.int16).astype(np.int64)
    pw = (re * re + im * im).astype(np.uint64).astype(np.uint32).view(np.int32)
    root = np.sqrt(pw.astype(np.float32).clip(0))
    m = (root * np.float32(10)).astype(np.float32)
    return np.where(pw < 0, 0, np.trunc(m)).astype(np.uint64)


def filter_sums(energy, g):
    """pow_spct of MFCC.C:136-162, bin by bin: sum over [lo, hi) of (E * tri / 100), every product and sum in u32"""
    out = np.zeros((energy.shape[0], 24), np.uint64)
    for h in range(24):
        acc = np.zeros(energy.shape[0], np.uint64)
        for k in range(g.lo[h], g.hi[h]):
            acc = (acc + ((energy[:, k] * g.w[h & 1][k]) & M32) // np.uint64(100)) & M32
        out[:, h] = acc
    return out


def log100(v):
    """(u32)(log(v) * 100) of MFCC.C:168 as the last L with thr[L] <= v; log(0) pinned to 0 (DESIGN §3)"""
    v = np.asarray(v, np.uint64)
    return np.where(v == 0, 0, np.searchsorted(THR, v, side="right") - 1).astype(np.int64)


def dct(lg, g):
    """MFCC.C:173-183: coefficient c = sum over filters i of (s32)lg[i] * dct[c][i] / 100, each term truncated toward
    zero, accumulated in an s16"""
    terms = _cdiv(lg[:, None, :] * g.dct[None, :, :], 100)
    return terms.sum(axis=2).astype(np.int16)


def coefficients(sums, g):
    """the 12 coefficients of frames with the given filter sums [n, 24]"""
    return dct(log100(sums), g)


def stages(cur, prv, mid, g, fft=None):
    """every stage of n frames: cur [n, frame] the frame's samples, prv [n, frame] the sample before each one, mid [n].
    Returns a dict of win [n, frame] s16, spec [n, n_fft] packed, mag / energy [n, bins], sums [n, 24], lg [n, 24],
    mfcc [n, 12] s16"""
    fft = fft or ob.port()
    win = windowed(cur, prv, mid, g.hamm)
    packed = np.zeros((cur.shape[0], g.n_fft), np.uint32)
    packed[:, :g.frame] = win.view(np.uint16)                            # fft_in[i] = *(u16 *)(dat_buf + i), zero padded
    spec = fft.fft_raw(packed) if g.n_fft == 1024 else fft.fft_raw_n(packed, g.n_fft)
    mag = magnitude(spec, g.bins)
    energy = (mag * mag) & M32                                           # frq_spct[i] *= frq_spct[i], u32
    sums = filter_sums(energy, g)
    lg = log100(sums)
    return dict(win=win, spec=spec, mag=mag, energy=energy, sums=sums, lg=lg, mfcc=dct(lg, g))


def segment_frames(pcm, seg, atap, g):
    """the frames get_mfcc reads from segments [start, end) of rows of pcm (start >= 1): (cur, prv, mid, row, frame)"""
    cur, prv, mid, rows, idx = [], [], [], [], []
    for b in range(pcm.shape[0]):
        st, en = int(seg[b, 0]), int(seg[b, 1])
        assert st >= 1, "segment_frames reads x[start - 1] from the row"
        for f in range(g.frames_of(en - st)):
            a = st + g.hop * f
            cur.append(pcm[b, a:a + g.frame])
            prv.append(pcm[b, a - 1:a - 1 + g.frame])
            mid.append(int(atap["mid_val"][b]))
            rows.append(b)
            idx.append(f)
    L = g.frame
    return (np.array(cur, np.uint16).reshape(-1, L), np.array(prv, np.uint16).reshape(-1, L), np.array(mid, np.int64),
            np.array(rows, np.int64), np.array(idx, np.int64))


def mfcc_batch(pcm, seg, atap, g, fft=None):
    """get_mfcc of one segment per row, through the stages: (ftr, sums [n_frames, 24], row of each frame)"""
    cur, prv, mid, rows, idx = segment_frames(pcm, seg, atap, g)
    ftr = np.zeros(pcm.shape[0], ob.FTR_DTYPE)
    for b in range(pcm.shape[0]):
        ftr["frm_num"][b] = g.frames_of(int(seg[b, 1]) - int(seg[b, 0]))
    if len(rows) == 0:
        return ftr, np.zeros((0, 24), np.uint64), rows
    st = stages(cur, prv, mid, g, fft)
    for m, b, f in zip(st["mfcc"], rows, idx):
        ftr["mfcc_dat"][b][12 * f:12 * f + 12] = m
    return ftr, st["sums"], rows


def exposure(sums, g):
    """[n, 24, 2] bool: frame i exposes filter h upwards (index 0) / downwards (index 1) when moving that filter's sum
    by +1 / -1, all else equal, changes its 12 coefficients. Moves stay inside u32 (no wrap past 0 or 2^32 - 1)"""
    base = coefficients(sums, g)
    out = np.zeros(sums.shape + (2,), bool)
    for h in range(24):
        for j, d in enumerate((1, -1)):
            s = sums.astype(np.int64).copy()
            ok = (s[:, h] + d >= 0) & (s[:, h] + d <= 0xFFFFFFFF)
            s[:, h] = np.where(ok, s[:, h] + d, s[:, h])
            out[:, h, j] = ok & (coefficients(s.astype(np.uint64), g) != base).any(axis=1)
    return out


# ---- one-frame inputs that reach the sensitive regime of the filter sums --------------------------------------------
def _candidates(g, rng, n):
    """one-frame rows [n, frame + 1] (x[-1] first) near a mid_val: few samples off mid (most bins then hold 0 to a few
    units of energy), quiet noise of mid +- 1 .. 32, and quiet tones on filter edges, 16-bin lane boundaries and 4-bin
    groups; mid_val 0, 2 048, 65 535 and two others"""
    L = g.frame
    mid = rng.choice([0, 2048, 65535, 1000, 30000], n).astype(np.int64)
    x = np.repeat(mid[:, None], L + 1, 1)
    kind = np.arange(n) % 4
    for i in np.flatnonzero(kind < 2):                         # sparse: 1..5 samples off mid by up to +-60 (or +-8)
        k = int(rng.integers(1, 6))
        amp = 60 if kind[i] == 0 else 8
        x[i, rng.integers(0, L + 1, k)] += rng.integers(-amp, amp + 1, k)
    i3 = np.flatnonzero(kind == 2)                             # noise
    a = rng.choice([1, 2, 3, 4, 6, 8, 16, 32], len(i3))[:, None]
    x[i3] += rng.integers(0, 1 << 20, (len(i3), L + 1)) % (2 * a + 1) - a
    i4 = np.flatnonzero(kind == 3)                             # tones
    edges = sorted(set(g.lo + [h - 1 for h in g.hi] + list(range(0, g.bins, 16)) + list(range(3, g.bins, 4))))
    kb = rng.choice(edges, len(i4))[:, None] + rng.choice([-0.25, 0, 0.25], len(i4))[:, None]
    amp = rng.choice([1, 2, 3, 5, 8, 12, 20], len(i4))[:, None]
    x[i4] += np.round(amp * np.cos(2 * np.pi * kb * np.arange(L + 1) / g.n_fft + rng.random((len(i4), 1)) * 6.28)).astype(np.int64)
    return np.clip(x, 0, 65535).astype(np.uint16), mid


@functools.lru_cache(maxsize=None)
def exposing_frames(g, seed=0x6D46, per_pair=6, n_pool=8000):
    """one-frame rows (x[-1] first) and their mid_vals, selected from a seeded pool so that every (filter, sign) is
    exposed by at least `per_pair` frames (greedy cover), plus every pool frame with a filter sum in 1 .. 99, frames
    that sit exactly on a threshold and one below it, frames whose sums mix 0 and nonzero, and all-zero frames (every
    sample at mid_val) for mid_val 0, 2 048 and 65 535. Returns (rows [n, frame + 1] u16, mid [n], stages of the rows)"""
    rng = np.random.default_rng(seed)
    rows, mid = _candidates(g, rng, n_pool)
    st = stages(rows[:, 1:], rows[:, :-1], mid, g)
    ex = exposure(st["sums"], g).reshape(len(rows), 48)
    need = np.full(48, per_pair)
    pick = []
    while (need > 0).any():
        gain = ex[:, need > 0].sum(axis=1)
        gain[pick] = 0
        i = int(np.argmax(gain))
        assert gain[i] > 0, "the pool exposes (filter, sign) %s fewer than %d times" % (np.flatnonzero(need > 0), per_pair)
        pick.append(i)
        need -= ex[i]
    s = st["sums"].astype(np.int64)
    small = np.flatnonzero(((s >= 1) & (s <= 99)).any(axis=1))
    on_thr = np.flatnonzero(np.isin(s, THR[100:].astype(np.int64)).any(axis=1))[:8]       # sum = thr[L], L >= 100
    below = np.flatnonzero(np.isin(s, THR[100:].astype(np.int64) - 1).any(axis=1))[:8]    # sum = thr[L] - 1
    mixed = np.flatnonzero((s == 0).any(axis=1) & (s > 0).any(axis=1))[:8]
    sel = list(dict.fromkeys(pick + small.tolist() + on_thr.tolist() + below.tolist() + mixed.tolist()))
    zero = np.repeat(np.array([[0], [2048], [65535]], np.uint16), g.frame + 1, 1)
    rows = np.concatenate([rows[sel], zero])
    mid = np.concatenate([mid[sel], [0, 2048, 65535]])
    return rows, mid, stages(rows[:, 1:], rows[:, :-1], mid, g)
