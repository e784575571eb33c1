"""Checkers of the long-form calls (include/sr_long.h, TEST INFRASTRUCTURE):
  LongOracle      -- ctypes binding of oracle/_build/liboracle_long.so, built by __graft_entry__.build() from
                     tests/oracle_long.c: the long-form VAD (VAD.C:97-218 without max_vc_con, u32 length)
  recognise_long  -- sr_recognise_long_batch composed from that VAD and the port's noise_atap, get_mfcc and dtw"""
import ctypes as C
import os

import numpy as np

from oracle_bind import ATAP_DTYPE, FTR_DTYPE, NULL, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LONG_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_long.so")
LONG_SEG_DTYPE = np.dtype([(k, "<u4") for k in ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")])


class LongOracle:
    name = "oracle-long"

    def __init__(self):
        self.lib = C.CDLL(LONG_SO)
        self.lib.sro_vad_long.restype = C.c_uint32

    def vad_long(self, pcm, atap, max_segs, lens=None, nthreads=8):
        """pcm [B, U], atap [B] -> (n_segs [B], seg [B, max_segs, 2]; slots past n_segs stay 0)"""
        pcm = np.ascontiguousarray(pcm, np.uint16)
        B, U = pcm.shape
        atap = np.ascontiguousarray(atap, ATAP_DTYPE).reshape(B)
        lens = None if lens is None else np.ascontiguousarray(lens, np.uint32)
        n = np.zeros(B, np.uint32)
        seg = np.zeros((B, max(max_segs, 1), 2), np.uint32)
        self.lib.sro_vad_long_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), _p(lens), _p(atap), C.c_uint32(max_segs),
                                    _p(n), _p(seg), C.c_int(nthreads))
        return n, seg[:, :max_segs]


def synth_long(B, U, seed):
    """B synthetic recordings of U samples with many words: 2-second utterances of sr_synth_pcm_host (300 ms of noise,
    then 3 words) back to back, each shifted to the DC level of its recording's first one, so that VAD finds the words"""
    import sr_b200
    n = -(-U // 16000)
    utt = sr_b200.synth_pcm_host(B * n, 16000, seed, 3).reshape(B, n, 16000).astype(np.int32)
    dc = utt[:, :, :2400].mean(axis=2).round().astype(np.int32)
    utt += (dc[:, :1] - dc)[:, :, None]
    return np.ascontiguousarray(np.clip(utt, 0, 4095).astype(np.uint16).reshape(B, n * 16000)[:, :U])


def long_oracle():
    return LongOracle()


def atap_long(port, pcm, n_len, lens=None, atap=None):
    """noise_atap over the first n_len samples of each recording; atap[b] untouched when n_len % 240 != 0 or n_len > lens[b]"""
    B, U = pcm.shape
    atap = np.zeros(B, ATAP_DTYPE) if atap is None else atap.copy()
    for b in range(B):
        if n_len <= (U if lens is None else int(lens[b])):
            atap[b] = port.noise_atap(np.ascontiguousarray(pcm[b]), n_len, atap[b:b + 1])[0]
    return atap


def recognise_long(lo, port, pcm, n_len, bank, n_slot, slot_stride, max_segs, lens=None, band_r=-1, geom_b=False,
                   atap=None, rows=None):
    """sr_recognise_long_batch from the oracles' stages: dict(atap, n_segs, segs [B, max_segs] LONG_SEG_DTYPE, zeros past
    n_segs). rows: recordings whose segments get records (None: all; the others' records stay zero)."""
    B, U = pcm.shape
    atap = atap_long(port, pcm, n_len, lens, atap)
    n, seg = lo.vad_long(pcm, atap, max_segs, lens)
    segs = np.zeros((B, max_segs), LONG_SEG_DTYPE)
    frame_len = 200 if geom_b else 160
    todo = []                                                # (b, k, start, end) with 1..119 frames
    for b in range(B) if rows is None else rows:
        for k in range(min(int(n[b]), max_segs)):
            st, en = int(seg[b, k, 0]), int(seg[b, k, 1])
            r = segs[b, k]
            r["start"], r["end"], r["best_idx"], r["best_dis"], r["cmd"] = st, en, 0, NULL, 0
            if en == NULL:
                r["status"] = 1                              # main.c:261-266
                continue
            F = (en - st - frame_len) // 80 + 1 if en - st >= frame_len else 0
            if 1 <= F <= 119:
                todo.append((b, k, st, en))
            else:
                r["status"] = 2                              # main.c:269-274 (over 119 frames: MFCC.C:103-107)
    if not todo:
        return dict(atap=atap, n_segs=n, segs=segs)
    L = max(en - st for _, _, st, en in todo)
    xs = np.zeros((len(todo), L + 1), np.uint16)             # [x[-1], samples]: x[-1] = mid_val at sample 0
    for i, (b, k, st, en) in enumerate(todo):
        xs[i, 0] = pcm[b, st - 1] if st else np.uint16(atap["mid_val"][b] & 0xFFFF)
        xs[i, 1:1 + en - st] = pcm[b, st:en]
    s2 = np.array([[1, 1 + en - st] for _, _, st, en in todo], np.uint32)
    at = atap[[b for b, _, _, _ in todo]]
    ftr = port.mfcc_geom_b_batch(xs, s2, at) if geom_b else port.mfcc_batch(xs, s2, at, nthreads=8)
    if n_slot:
        sc, _ = port.dtw_batch(ftr, bank, n_slot, slot_stride, check_sign=1, band_r=band_r, nthreads=8)
    for i, (b, k, st, en) in enumerate(todo):
        r = segs[b, k]
        r["frm_num"] = ftr["frm_num"][i]
        if ftr["frm_num"][i] == 0:
            r["status"] = 2
            continue
        r["status"] = 0
        if n_slot:
            j = int(np.argmin(sc[i]))                        # first of the minima: the strict '<' scan (main.c:285-289)
            if sc[i, j] != NULL:
                r["best_idx"], r["best_dis"], r["cmd"] = j, sc[i, j], j // 4
    return dict(atap=atap, n_segs=n, segs=segs)


def ftr_of_segments(port, pcm, atap, seg_list, geom_b=False):
    """get_mfcc of (b, start, end) segments with x[-1] of a segment at sample 0 pinned to mid_val: FTR_DTYPE [n]"""
    if not seg_list:
        return np.zeros(0, FTR_DTYPE)
    L = max(en - st for _, st, en in seg_list)
    xs = np.zeros((len(seg_list), L + 1), np.uint16)
    for i, (b, st, en) in enumerate(seg_list):
        xs[i, 0] = pcm[b, st - 1] if st else np.uint16(atap["mid_val"][b] & 0xFFFF)
        xs[i, 1:1 + en - st] = pcm[b, st:en]
    s2 = np.array([[1, 1 + en - st] for _, st, en in seg_list], np.uint32)
    at = atap[[b for b, _, _ in seg_list]]
    return port.mfcc_geom_b_batch(xs, s2, at) if geom_b else port.mfcc_batch(xs, s2, at, nthreads=8)
