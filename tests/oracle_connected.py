"""Checkers of the connected-word calls (TEST INFRASTRUCTURE):
  ConnectedOracle  -- ctypes binding of oracle/_build/liboracle_connected.so, built by __graft_entry__.build() from
                      tests/oracle_connected.c: the CPU restatement of sr_connected_batch
  mfcc_long        -- sr_mfcc_long_batch composed from an oracle's own get_mfcc, piece by piece
  recognise_connected -- sr_recognise_connected_batch composed from the oracle stages"""
import ctypes as C
import os

import numpy as np

from oracle_bind import ATAP_DTYPE, NULL, _p, pinned_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONNECTED_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_connected.so")
CONN_FRM_MAX = 818
WORD_DTYPE = np.dtype([(k, "<u4") for k in ("slot", "cmd", "segment", "start", "end", "dis")])


class ConnectedOracle:
    name = "oracle-connected"

    def __init__(self):
        self.lib = C.CDLL(CONNECTED_SO)

    def connected(self, feat, frm, bank, n_slot, slot_stride, penalty, max_words, nthreads=1):
        """feat [B, stride, 12] i16, frm [B] -> (words [B, max_words] WORD_DTYPE (zeros past n_words), n_words [B],
        total [B] u64)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm = np.ascontiguousarray(frm, np.uint32)
        bank = np.ascontiguousarray(bank, np.uint8) if n_slot else np.zeros(16, np.uint8)
        words = np.zeros((B, max_words), WORD_DTYPE)
        n_words, total = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
        self.lib.sro_connected_batch(_p(feat), _p(frm), C.c_uint32(stride), C.c_uint32(B), _p(bank), C.c_uint32(n_slot),
                                     C.c_uint32(slot_stride), C.c_uint32(penalty), C.c_uint32(max_words), _p(words),
                                     _p(n_words), _p(total), C.c_int(nthreads))
        return words, n_words, total


def connected():
    return ConnectedOracle()


def long_frames(st, en, U, frame_len):
    """the frame count of MFCC.C:102-107 without the vv_frm_max cap (0 for NULL, reversed or short segments)"""
    if st == NULL or en == NULL or en > U or st > en or en - st < frame_len:
        return 0
    return (en - st - frame_len) // 80 + 1


def mfcc_long(ora, pcm, seg2, atap, frm_cap, geom_b=False):
    """sr_mfcc_long_batch from an oracle's get_mfcc: each segment cut into pieces of <= 119 frames, piece k starting at
    sample start + 80*119*k, every piece a get_mfcc segment of pinned_rows ([mid_val, row...], segments shifted by +1), so
    x[-1] is mid_val only for a piece at sample 0. Returns (feat [B, frm_cap, 12] i16, zeros where nothing is written,
    frm_num [B])"""
    B, U = pcm.shape
    seg2 = np.asarray(seg2, np.uint32).reshape(B, 2)
    frame_len = 200 if geom_b else 160
    feat = np.zeros((B, frm_cap, 12), np.int16)
    frm = np.zeros(B, np.uint32)
    pieces = []
    for b in range(B):
        st, en = int(seg2[b, 0]), int(seg2[b, 1])
        F = long_frames(st, en, U, frame_len)
        if F > frm_cap:
            F = 0
        frm[b] = F
        for f0 in range(0, F, 119):
            nf = min(119, F - f0)
            ps = st + 80 * f0
            pieces.append((b, f0, nf, ps, ps + 80 * (nf - 1) + frame_len))
    if pieces:
        idx = np.array([p[0] for p in pieces])
        rows = pinned_rows(pcm[idx], atap[idx])
        seg = np.array([[p[3] + 1, p[4] + 1] for p in pieces], np.uint32)
        f = ora.mfcc_geom_b_batch(rows, seg, atap[idx]) if geom_b else ora.mfcc_batch(rows, seg, atap[idx])
        for q, (b, f0, nf, _, _) in enumerate(pieces):
            assert int(f["frm_num"][q]) == nf
            feat[b, f0:f0 + nf] = f["mfcc_dat"][q][: nf * 12].reshape(nf, 12)
    return feat, frm


def recognise_connected(ora, co, pcm, n_len, bank, n_slot, slot_stride, penalty, max_words, geom_b=False, atap0=None):
    """sr_recognise_connected_batch composed from the oracle stages: noise_atap and VAD per row, mfcc_long of every segment
    at frm_cap = 818, the decoder on each segment with frames, the words joined in segment order (segment set), total the
    saturating sum, status from segment 0. atap0: the atap records noise_atap starts from (it leaves them untouched when
    n_len % 240 != 0; default zeros). Returns a dict of the sr_conn_out fields (words zero past n_words)"""
    B, U = pcm.shape
    out = dict(atap=np.zeros(B, ATAP_DTYPE), seg_off=np.zeros((B, 3, 2), np.uint32), frm_num=np.zeros((B, 3), np.uint32),
               n_words=np.zeros(B, np.uint32), words=np.zeros((B, max_words), WORD_DTYPE), total=np.zeros(B, np.uint64),
               status=np.zeros(B, np.uint8))
    for b in range(B):
        out["atap"][b] = ora.noise_atap(pcm[b], n_len, None if atap0 is None else atap0[b:b + 1])[0]
        out["seg_off"][b] = ora.vad(pcm[b], U, out["atap"][b:b + 1]).reshape(3, 2)
    feats = []
    for k in range(3):
        f, n = mfcc_long(ora, pcm, out["seg_off"][:, k, :], out["atap"], CONN_FRM_MAX, geom_b)
        feats.append(f)
        out["frm_num"][:, k] = n
    for b in range(B):
        cnt, tot = 0, 0
        for k in range(3):
            n = int(out["frm_num"][b, k])
            if n == 0:
                continue
            w, nw, t = co.connected(feats[k][b:b + 1, :max(n, 1)], np.array([n], np.uint32), bank, n_slot, slot_stride,
                                    penalty, int(n))
            nw = int(nw[0])
            for q in range(nw):
                if cnt + q < max_words:
                    out["words"][b, cnt + q] = w[0, q]
                    out["words"][b, cnt + q]["segment"] = k
            cnt += nw
            tot = min(tot + int(t[0]), 2 ** 64 - 1)
        out["n_words"][b], out["total"][b] = cnt, tot
        out["status"][b] = 1 if out["seg_off"][b, 0, 1] == NULL else 2 if out["frm_num"][b, 0] == 0 else 0
    return out
