"""The oracle of SR_DTW_LIFTER (TEST INFRASTRUCTURE, CPU only): the transform L as a plain numpy function, and the
recognition oracles under the bit composed from the existing ones by its defining rule -- every matcher scores (x, y)
with the bit exactly as it scores (L(x), L(y)) without it. No DP code is restated here: the inputs and a copy of the bank
are liftered and handed to oracle_ext's matchers."""
import numpy as np

import oracle_ext as ox
from oracle_bind import FTR_DTYPE, NULL

LIFTER = 1 << 13               # SR_DTW_LIFTER


def lifter(rows):
    """SR_DTW_LIFTER's transform of s16 cepstral rows (any shape whose last axis is a multiple of 12, coefficient c of a
    row being c_{c+1}): a' = sat16(trunc(a * W / 16)), W = round(4 (1 + 6 sin(pi k / 12))) for k = 1..12"""
    w = np.round(4 * (1 + 6 * np.sin(np.pi * np.arange(1, 13) / 12))).astype(np.int64)
    a = np.asarray(rows)
    p = a.reshape(-1, 12).astype(np.int64) * w
    q = np.sign(p) * (np.abs(p) // 16)                                   # C division: truncation toward zero
    return np.clip(q, -32768, 32767).astype(np.int16).reshape(a.shape)


def lifter_ftr(ftr):
    """a copy of feature structs with every one of their 119 rows liftered"""
    out = np.array(ftr, FTR_DTYPE, copy=True)
    out["mfcc_dat"] = lifter(out["mfcc_dat"])
    return out


def lifter_bank(bank, n_slot, slot_stride=4096):
    """a copy of a flash-layout bank with every row of its first n_slot slots liftered, headers as they are"""
    out = np.array(bank, np.uint8, copy=True).reshape(-1)
    if n_slot:
        slots = out[:n_slot * slot_stride].reshape(n_slot, slot_stride)
        f = np.ascontiguousarray(slots[:, :FTR_DTYPE.itemsize]).view(FTR_DTYPE).reshape(n_slot)
        slots[:, :FTR_DTYPE.itemsize] = lifter_ftr(f).view(np.uint8).reshape(n_slot, FTR_DTYPE.itemsize)
    return out.reshape(np.shape(bank))


def match_scores(ftr, bank, n_slot, flags, r, slot_stride=4096):
    """oracle_ext.match_scores under the matcher (flags, r), SR_DTW_LIFTER included: with the bit, the same matcher on the
    liftered inputs against a liftered copy of the bank"""
    if flags & LIFTER:
        return ox.match_scores(lifter_ftr(ftr), lifter_bank(bank, n_slot, slot_stride), n_slot, flags & ~LIFTER, r,
                               slot_stride)
    return ox.match_scores(ftr, bank, n_slot, flags, r, slot_stride)


def compose_recognise(front, bank, T, flags, r):
    """oracle_ext.compose_recognise under the matcher (flags, r), SR_DTW_LIFTER included; the features the call returns
    are the front end's, not liftered"""
    if not flags & LIFTER:
        return ox.compose_recognise(front, bank, T, flags, r)
    out = ox.compose_recognise(dict(front, ftr=lifter_ftr(front["ftr"])), lifter_bank(bank, T), T, flags & ~LIFTER, r)
    out["ftr"] = np.array(front["ftr"], copy=True)
    return out


def recognise_long(lo, port, pcm, n_len, bank, n_slot, slot_stride, max_segs, lens=None, match=(0, 0)):
    """oracle_ext.recognise_long under the matcher match = (flags, r), SR_DTW_LIFTER included: its segments and statuses,
    then each SR_ST_OK segment scored by match_scores and decided by the strict '<' first-wins argmin (main.c:285-289)"""
    w = ox.recognise_long(lo, port, pcm, n_len, bank, 0, slot_stride, max_segs, lens)
    segs = w["segs"]
    todo = [(b, k) for b in range(len(segs)) for k in range(min(int(w["n_segs"][b]), max_segs)) if segs[b, k]["status"] == 0]
    if todo and n_slot:
        ftr = ox.ftr_of_segments(port, pcm, w["atap"], [(b, int(segs[b, k]["start"]), int(segs[b, k]["end"])) for b, k in todo])
        sc = match_scores(ftr, bank, n_slot, *match, slot_stride=slot_stride)
        for i, (b, k) in enumerate(todo):
            j = int(np.argmin(sc[i]))
            if sc[i, j] != NULL:
                segs[b, k]["best_idx"], segs[b, k]["best_dis"], segs[b, k]["cmd"] = j, sc[i, j], j // 4
    return w
