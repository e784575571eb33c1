"""Checkers of the extension calls (TEST INFRASTRUCTURE):
  ctypes bindings of oracle/_build/liboracle_ext.so, built by __graft_entry__.build() from tests/oracle_ext/*.c -- the CPU
  restatements of the alignment calls, the connected-word decoder, the grammar decoder (capture and segment-table forms),
  the long-form VAD, the symmetric P = 1 matcher and the banded DP without the 2:1 guard;
  recognition's template scan under every matcher (match_scores) and the end-to-end calls composed from them and the
  oracle port's stages (compose_recognise, mfcc_long, recognise_connected, recognise_connected_grammar, recognise_long,
  recognise_long_grammar); a call's records under a decision rule (under_rule, long_under_rule); and the recordings and
  banks the tests share."""
import ctypes as C
import functools
import os

import numpy as np

from oracle_bind import ATAP_DTYPE, FTR_DTYPE, NULL, PortOracle, _p, segment_rows
from refs import NTHREADS, decide

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_ext.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")
PATH_MAX = 237
CONN_FRM_MAX = 818
SEG_NONE = 0xFFFFFFFF
WORD_DTYPE = np.dtype([(k, "<u4") for k in ("slot", "cmd", "segment", "start", "end", "dis")])
LONG_SEG_DTYPE = np.dtype([(k, "<u4") for k in ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")])


@functools.cache
def _lib():
    lib = C.CDLL(EXT_SO)
    lib.sro_rate_d.restype = C.c_int64
    lib.sro_rate_d.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    lib.sro_sym_g.restype = C.c_uint64
    lib.sro_sym_g.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return lib


def _bank(bank, n_slot):
    return np.ascontiguousarray(bank, np.uint8) if n_slot else np.zeros(16, np.uint8)


def _arcs(g):
    n_states, final_mask, arcs = g
    a = np.array(arcs, np.uint32).reshape(-1, 3) if arcs else np.zeros((1, 3), np.uint32)
    return int(n_states), int(final_mask), len(arcs), np.ascontiguousarray(a)


def _decoded(B, max_words, call):
    """words [B, max_words] WORD_DTYPE (zeros past n_words), n_words [B], total [B] u64, filled by call(words, n, total)"""
    words = np.zeros((B, max_words), WORD_DTYPE)
    n_words, total = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    call(_p(words), _p(n_words), _p(total))
    return words, n_words, total


class AlignOracle:
    """sr_dtw_path_batch and sr_average_bank (tests/oracle_ext/align.c)"""

    def dtw_path(self, fin, fmdl, r, nthreads=1, with_path=True):
        """n pairs (fin[p], fmdl[p]) -> (dis [n], path [n, 237, 2] or None, path_len [n] or None)"""
        fin, fmdl = np.ascontiguousarray(fin, FTR_DTYPE), np.ascontiguousarray(fmdl, FTR_DTYPE)
        n = len(fin)
        assert len(fmdl) == n
        dis = np.zeros(n, np.uint32)
        path = np.zeros((n, PATH_MAX, 2), np.uint8) if with_path else None
        plen = np.zeros(n, np.uint32) if with_path else None
        _lib().sro_dtw_path_batch(_p(fin), _p(fmdl), C.c_uint32(n), C.c_int(min(r, 2 ** 31 - 1)), _p(path), _p(plen),
                                  _p(dis), C.c_int(nthreads))
        return dis, path, plen

    def average_bank(self, bank, slot_stride, K, r, iters, nthreads=1):
        """bank [G*K, slot_stride] u8 -> (bank_out of the same shape, score [G, K], anchor [G])"""
        bank = np.ascontiguousarray(bank, np.uint8).reshape(-1, slot_stride)
        G = bank.shape[0] // K
        out = np.zeros_like(bank)
        score, anchor = np.zeros((G, K), np.uint32), np.zeros(G, np.uint32)
        _lib().sro_average_bank(_p(bank), C.c_uint32(slot_stride), C.c_uint32(K), C.c_uint32(G), C.c_int(r),
                                C.c_uint32(iters), _p(out), _p(score), _p(anchor), C.c_int(nthreads))
        return out, score, anchor


class ConnectedOracle:
    """sr_connected_batch (tests/oracle_ext/connected.c)"""

    def connected(self, feat, frm, bank, n_slot, slot_stride, penalty, max_words, nthreads=1):
        """feat [B, stride, 12] i16, frm [B] -> (words [B, max_words] WORD_DTYPE (zeros past n_words), n_words [B],
        total [B] u64)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm, bank = np.ascontiguousarray(frm, np.uint32), _bank(bank, n_slot)
        return _decoded(B, max_words, lambda w, n, t: _lib().sro_connected_batch(
            _p(feat), _p(frm), C.c_uint32(stride), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
            C.c_uint32(penalty), C.c_uint32(max_words), w, n, t, C.c_int(nthreads)))


class GrammarOracle:
    """sr_connected_grammar_batch (the capture form of tests/oracle_ext/long_grammar.c)"""

    def decode(self, feat, frm, bank, n_slot, slot_stride, grammar, penalty, max_words, seg=None, nthreads=1):
        """feat [B, stride, 12] i16, frm [B], grammar (n_states, final_mask, [(from, to, cmd_mask), ...]), seg [B, 3]
        segment first frames (SEG_NONE: no frames) or None -> (words [B, max_words] WORD_DTYPE (zeros past n_words),
        n_words [B], total [B] u64)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm, bank = np.ascontiguousarray(frm, np.uint32), _bank(bank, n_slot)
        S, F, n_arcs, arcs = _arcs(grammar)
        seg = None if seg is None else np.ascontiguousarray(seg, np.uint32).reshape(B, 3)
        return _decoded(B, max_words, lambda w, n, t: _lib().sro_grammar_batch(
            _p(feat), _p(frm), C.c_uint32(stride), _p(seg), C.c_uint32(B), _p(bank), C.c_uint32(n_slot),
            C.c_uint32(slot_stride), C.c_uint32(S), C.c_uint32(F), C.c_uint32(n_arcs), _p(arcs), C.c_uint32(penalty),
            C.c_uint32(max_words), w, n, t, C.c_int(nthreads)))


class LongGrammarOracle:
    """sr_connected_grammar_segs_batch (tests/oracle_ext/long_grammar.c)"""

    def decode_segs(self, feat, seq_seg, seg_frm, bank, n_slot, slot_stride, grammar, penalty, max_words, nthreads=8):
        """feat [rows, 12] i16, seq_seg [B+1], seg_frm [n_seg], grammar (n_states, final_mask, [(from, to, cmd_mask), ...])
        -> (words [B, max_words] WORD_DTYPE (zeros past n_words), n_words [B], total [B] u64)"""
        feat = np.ascontiguousarray(feat, np.int16).reshape(-1, 12)
        if feat.shape[0] == 0:
            feat = np.zeros((1, 12), np.int16)
        seq_seg = np.ascontiguousarray(seq_seg, np.uint32)
        seg_frm = np.ascontiguousarray(seg_frm, np.uint32)
        if seg_frm.size == 0:
            seg_frm = np.zeros(1, np.uint32)
        B = len(seq_seg) - 1
        bank = _bank(bank, n_slot)
        S, F, n_arcs, arcs = _arcs(grammar)
        return _decoded(B, max_words, lambda w, n, t: _lib().sro_long_grammar_batch(
            _p(feat), _p(seq_seg), _p(seg_frm), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
            C.c_uint32(S), C.c_uint32(F), C.c_uint32(n_arcs), _p(arcs), C.c_uint32(penalty), C.c_uint32(max_words), w, n,
            t, C.c_int(nthreads)))


class LongOracle:
    """sr_vad_long_batch: the long-form VAD, VAD.C:97-218 without max_vc_con, u32 length (tests/oracle_ext/long.c)"""

    def vad_long(self, pcm, atap, max_segs, lens=None, nthreads=8):
        """pcm [B, U], atap [B] -> (n_segs [B], seg [B, max_segs, 2]; slots past n_segs stay 0)"""
        pcm = np.ascontiguousarray(pcm, np.uint16)
        B, U = pcm.shape
        atap = np.ascontiguousarray(atap, ATAP_DTYPE).reshape(B)
        lens = None if lens is None else np.ascontiguousarray(lens, np.uint32)
        n = np.zeros(B, np.uint32)
        seg = np.zeros((B, max(max_segs, 1), 2), np.uint32)
        _lib().sro_vad_long_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), _p(lens), _p(atap), C.c_uint32(max_segs), _p(n),
                                  _p(seg), C.c_int(nthreads))
        return n, seg[:, :max_segs]


class _BankScores:
    """score [B, n_slot] of FTR_DTYPE inputs against a bank of n_slot slots of slot_stride bytes (sro_bank_scores)"""
    batch = None

    def dtw_batch(self, ftr_in, bank, n_slot, slot_stride, check_sign=0, band_r=0, nthreads=8):
        ftr_in = np.ascontiguousarray(ftr_in, FTR_DTYPE)
        bank = np.ascontiguousarray(bank).view(np.uint8)
        B = ftr_in.shape[0]
        score = np.zeros((B, n_slot), np.uint32)
        if B and n_slot:
            getattr(_lib(), self.batch)(_p(ftr_in), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
                                        C.c_int(check_sign), C.c_int(band_r), _p(score), C.c_int(nthreads))
        return score


class SymOracle(_BankScores):
    """SR_DTW_SYM_P1: Sakoe & Chiba's symmetric P = 1 DP over SR_DTW_BAND's band (tests/oracle_ext/sym.c)"""
    batch = "sro_sym_batch"

    def g(self, x, y, r):
        """g(I-1, M-1) of rows x [I, 12] against y [M, 12] (1..119 rows each) at radius r, or None when unreachable"""
        x, y = np.ascontiguousarray(x, np.int16), np.ascontiguousarray(y, np.int16)
        v = _lib().sro_sym_g(_p(x), len(x), _p(y), len(y), int(min(r, 118)))
        return None if v == 2 ** 64 - 1 else int(v)


class RateOracle(_BankScores):
    """SR_DTW_BAND | SR_DTW_ANY_RATE: the band DP over every cell with the band test and no guard (tests/oracle_ext/rate.c)"""
    batch = "sro_rate_batch"

    def d(self, x, y, r):
        """D(I-1, M-1) of rows x [I, 12] against y [M, 12] (1..119 rows each) at radius r, or None when unreachable"""
        x, y = np.ascontiguousarray(x, np.int16), np.ascontiguousarray(y, np.int16)
        v = _lib().sro_rate_d(_p(x), len(x), _p(y), len(y), int(min(r, 118)))
        return None if v == 2 ** 63 - 1 else int(v)


def align():
    return AlignOracle()


def connected():
    return ConnectedOracle()


def grammar():
    return GrammarOracle()


def long_grammar():
    return LongGrammarOracle()


def long_oracle():
    return LongOracle()


def sym_oracle():
    return SymOracle()


def rate_oracle():
    return RateOracle()


# ---- features ---------------------------------------------------------------------------------------------------------
def long_frames(st, en, U, frame_len):
    """the frame count of MFCC.C:102-107 without the vv_frm_max cap (0 for NULL, reversed or short segments)"""
    if st == NULL or en == NULL or en > U or st > en or en - st < frame_len:
        return 0
    return (en - st - frame_len) // 80 + 1


def ftr_of_segments(ora, pcm, atap, seg_list, geom_b=False):
    """get_mfcc of (b, start, end) segments with x[-1] of a segment at sample 0 pinned to mid_val: FTR_DTYPE [n]"""
    if not seg_list:
        return np.zeros(0, FTR_DTYPE)
    rows, s2 = segment_rows(pcm, atap, seg_list)
    at = atap[[b for b, _, _ in seg_list]]
    return ora.mfcc_geom_b_batch(rows, s2, at) if geom_b else ora.mfcc_batch(rows, s2, at, nthreads=8)


def piece_features(ora, pcm, atap, segs, geom_b=False):
    """sr_mfcc_long_batch's features of (b, start, F) segments of F frames from an oracle's get_mfcc, piece by piece:
    piece k of a segment has <= 119 frames, starts at sample start + 80*119*k and reads its real preceding sample (mid_val
    at sample 0). Returns [(b, first frame, rows [nf, 12] i16)], one per piece, in segment order"""
    frame_len = 200 if geom_b else 160
    pieces = [(b, f0, min(119, F - f0), st + 80 * f0) for b, st, F in segs for f0 in range(0, F, 119)]
    f = ftr_of_segments(ora, pcm, atap, [(b, ps, ps + 80 * (nf - 1) + frame_len) for b, _, nf, ps in pieces], geom_b)
    out = []
    for q, (b, f0, nf, _) in enumerate(pieces):
        assert int(f["frm_num"][q]) == nf
        out.append((b, f0, f["mfcc_dat"][q][: nf * 12].reshape(nf, 12)))
    return out


def mfcc_long(ora, pcm, seg2, atap, frm_cap, geom_b=False):
    """sr_mfcc_long_batch from an oracle's get_mfcc (piece_features). Returns (feat [B, frm_cap, 12] i16, zeros where
    nothing is written, frm_num [B])"""
    B, U = pcm.shape
    seg2 = np.asarray(seg2, np.uint32).reshape(B, 2)
    feat = np.zeros((B, frm_cap, 12), np.int16)
    frm = np.array([long_frames(int(st), int(en), U, 200 if geom_b else 160) for st, en in seg2], np.int64)
    frm = np.where(frm > frm_cap, 0, frm).astype(np.uint32)
    for b, f0, rows in piece_features(ora, pcm, atap, [(b, int(seg2[b, 0]), int(frm[b])) for b in range(B)], geom_b):
        feat[b, f0:f0 + len(rows)] = rows
    return feat, frm


def atap_long(port, pcm, n_len, lens=None, atap=None):
    """noise_atap over the first n_len samples of each recording; atap[b] untouched when n_len % 240 != 0 or n_len > lens[b]"""
    B, U = pcm.shape
    atap = np.zeros(B, ATAP_DTYPE) if atap is None else atap.copy()
    for b in range(B):
        if n_len <= (U if lens is None else int(lens[b])):
            atap[b] = port.noise_atap(np.ascontiguousarray(pcm[b]), n_len, atap[b:b + 1])[0]
    return atap


def _front_end(ora, pcm, n_len, atap0, geom_b):
    """noise_atap and VAD per capture, mfcc_long of every segment at frm_cap = 818: (atap, seg_off, frm_num, feats per
    segment, status from segment 0)"""
    B, U = pcm.shape
    atap, seg_off = np.zeros(B, ATAP_DTYPE), np.zeros((B, 3, 2), np.uint32)
    for b in range(B):
        atap[b] = ora.noise_atap(pcm[b], n_len, None if atap0 is None else atap0[b:b + 1])[0]
        seg_off[b] = ora.vad(pcm[b], U, atap[b:b + 1]).reshape(3, 2)
    feats, frm_num = zip(*(mfcc_long(ora, pcm, seg_off[:, k, :], atap, CONN_FRM_MAX, geom_b) for k in range(3)))
    frm_num = np.stack(frm_num, axis=1)
    status = np.where(seg_off[:, 0, 1] == NULL, 1, np.where(frm_num[:, 0] == 0, 2, 0)).astype(np.uint8)
    return dict(atap=atap, seg_off=seg_off, frm_num=frm_num, status=status), feats


# ---- the composed calls ---------------------------------------------------------------------------------------------------
def match_scores(ftr, bank, n_slot, flags, r, slot_stride=4096):
    """score [B, n_slot] of recognition's template scan under the matcher set by sr_set_match(flags, r), with the
    save_sign check: the port's greedy walk (flags 0) and SR_DTW_BAND DP, tests/oracle_ext/rate.c for SR_DTW_BAND |
    SR_DTW_ANY_RATE, tests/oracle_ext/sym.c for SR_DTW_SYM_P1"""
    import sr_b200
    if flags == sr_b200.DTW_SYM_P1:
        return sym_oracle().dtw_batch(ftr, bank, n_slot, slot_stride, check_sign=1, band_r=r, nthreads=NTHREADS)
    if flags == sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE:
        return rate_oracle().dtw_batch(ftr, bank, n_slot, slot_stride, check_sign=1, band_r=r, nthreads=NTHREADS)
    return PortOracle().dtw_batch(ftr, bank, n_slot, slot_stride, check_sign=1, band_r=r if flags else -1,
                                  nthreads=NTHREADS)[0]


def compose_recognise(front, bank, T, flags, r):
    """sr_recognise_batch under the matcher (flags, r) from a front end (oracle_bind.recognise_pinned's atap, seg_off,
    ftr and status): match_scores on the OK rows, the strict '<' first-wins argmin (main.c:276-294), cmd = idx / 4"""
    out = {k: front[k].copy() for k in ("atap", "seg_off", "ftr", "status")}
    B = len(out["status"])
    out["score"] = np.full((B, T), NULL, np.uint32)
    out["best_idx"], out["best_dis"], out["cmd"] = np.zeros(B, np.uint32), np.full(B, NULL, np.uint32), np.zeros(B, np.uint32)
    good = out["status"] == 0
    sc = match_scores(out["ftr"][good], bank, T, flags, r)
    out["score"][good] = sc
    i = np.argmin(sc, axis=1)                # first of the minima == the strict '<' scan from DIS_ERR
    out["best_idx"][good] = i
    out["best_dis"][good] = sc[np.arange(len(i)), i]
    out["cmd"][good] = i // 4
    return out



def under_rule(off, k, q):
    """what a recognition call writes under SR_DTW_KNN(k) | SR_DTW_REJECT(q), from the same call without a rule (off):
    refs.decide on the scores of its SR_ST_OK rows"""
    out = {key: np.array(v, copy=True) for key, v in off.items()}
    ok = np.flatnonzero(np.asarray(off["status"]) == 0)
    if len(ok) and np.asarray(off["score"]).shape[1]:
        idx, dis, cmd, rej = decide(np.asarray(off["score"])[ok], k, q)
        out["best_idx"][ok], out["best_dis"][ok], out["cmd"][ok] = idx, dis, cmd
        out["status"][ok] = np.where(rej, 3, 0)                            # SR_ST_REJECT, SR_ST_OK
    return out

def recognise_connected(ora, co, pcm, n_len, bank, n_slot, slot_stride, penalty, max_words, geom_b=False, atap0=None):
    """sr_recognise_connected_batch composed from the oracle stages: noise_atap and VAD per row, mfcc_long of every segment
    at frm_cap = 818, the decoder on each segment with frames, the words joined in segment order (segment set), total the
    saturating sum, status from segment 0. atap0: the atap records noise_atap starts from (it leaves them untouched when
    n_len % 240 != 0; default zeros). Returns a dict of the sr_conn_out fields (words zero past n_words)"""
    B = pcm.shape[0]
    out, feats = _front_end(ora, pcm, n_len, atap0, geom_b)
    out.update(n_words=np.zeros(B, np.uint32), words=np.zeros((B, max_words), WORD_DTYPE), total=np.zeros(B, np.uint64))
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
    return out


def recognise_connected_grammar(ora, go, pcm, n_len, bank, n_slot, slot_stride, grammar_, penalty, max_words, geom_b=False,
                                atap0=None, nthreads=1):
    """sr_recognise_connected_grammar_batch composed from the oracle stages: noise_atap and VAD per row, mfcc_long of every
    segment at frm_cap = 818, each capture's segments with frames back to back as one sequence decoded under the grammar
    with its segment table, status from segment 0. Returns a dict of the sr_conn_out fields (words zero past n_words)"""
    B = pcm.shape[0]
    out, feats = _front_end(ora, pcm, n_len, atap0, geom_b)
    x = np.zeros((B, CONN_FRM_MAX, 12), np.int16)
    N = np.zeros(B, np.uint32)
    seg = np.full((B, 3), SEG_NONE, np.uint32)
    for b in range(B):
        for k in range(3):
            n = int(out["frm_num"][b, k])
            if n:
                seg[b, k] = N[b]
                x[b, N[b]:N[b] + n] = feats[k][b, :n]
                N[b] += n
    out["words"], out["n_words"], out["total"] = go.decode(x, N, bank, n_slot, slot_stride, grammar_, penalty, max_words,
                                                           seg=seg, nthreads=nthreads)
    return out


def recognise_long(lo, port, pcm, n_len, bank, n_slot, slot_stride, max_segs, lens=None, match=(0, 0), geom_b=False,
                   atap=None, rows=None):
    """sr_recognise_long_batch from the oracles' stages: dict(atap, n_segs, segs [B, max_segs] LONG_SEG_DTYPE, zeros past
    n_segs), each segment scored by match_scores under the matcher match = (flags, r). rows: recordings whose segments
    get records (None: all; the others' records stay zero)."""
    B, U = pcm.shape
    atap = atap_long(port, pcm, n_len, lens, atap)
    n, seg = lo.vad_long(pcm, atap, max_segs, lens)
    segs = np.zeros((B, max_segs), LONG_SEG_DTYPE)
    todo = []                                                # (b, k, start, end) with 1..119 frames
    for b in range(B) if rows is None else rows:
        for k in range(min(int(n[b]), max_segs)):
            st, en = int(seg[b, k, 0]), int(seg[b, k, 1])
            r = segs[b, k]
            r["start"], r["end"], r["best_idx"], r["best_dis"], r["cmd"] = st, en, 0, NULL, 0
            if en == NULL:
                r["status"] = 1                              # main.c:261-266
            elif 1 <= long_frames(st, en, U, 200 if geom_b else 160) <= 119:
                todo.append((b, k, st, en))
            else:
                r["status"] = 2                              # main.c:269-274 (over 119 frames: MFCC.C:103-107)
    if not todo:
        return dict(atap=atap, n_segs=n, segs=segs)
    ftr = ftr_of_segments(port, pcm, atap, [(b, st, en) for b, _, st, en in todo], geom_b)
    if n_slot:
        sc = match_scores(ftr, bank, n_slot, *match, slot_stride=slot_stride)
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



def long_under_rule(off, pcm, n_len, lens, bank, n_slot, match, k, q, scores=match_scores):
    """what sr_recognise_long_batch writes under SR_DTW_KNN(k) | SR_DTW_REJECT(q) and the matcher match = (flags, r), from
    the same call's records without a rule (off): refs.decide on the oracles' scores of each SR_ST_OK segment (scores:
    the matcher's oracle, e.g. lifter_ref.match_scores for flags with SR_DTW_LIFTER)"""
    port = PortOracle()
    w = recognise_long(long_oracle(), port, pcm, n_len, bank, 0, 4096, off["segs"].shape[1], lens)
    segs = off["segs"].copy()
    todo = [(b, j) for b in range(len(segs)) for j in range(min(int(off["n_segs"][b]), segs.shape[1]))
            if segs[b, j]["status"] == 0]
    if todo:
        ftr = ftr_of_segments(port, pcm, w["atap"], [(b, int(segs[b, j]["start"]), int(segs[b, j]["end"])) for b, j in todo])
        idx, dis, cmd, rej = decide(scores(ftr, bank, n_slot, *match), k, q)
        for i, (b, j) in enumerate(todo):
            r = segs[b, j]
            r["best_idx"], r["best_dis"], r["cmd"], r["status"] = idx[i], dis[i], cmd[i], 3 if rej[i] else 0
    return dict(off, segs=segs)

def recognise_long_grammar(lo, port, lg, pcm, n_len, bank, n_slot, slot_stride, grammar, penalty, max_segs, max_words,
                           lens=None, geom_b=False, atap=None):
    """sr_recognise_long_grammar_batch from the oracles' stages: the long-form VAD of every segment, each decodable one's
    features, one decode per recording over its flat segment table. Returns a dict of the sr_long_gram_out fields (records
    past n_segs / n_words zero)"""
    B, U = pcm.shape
    atap = atap_long(port, pcm, n_len, lens, atap)
    n, _ = lo.vad_long(pcm, atap, 0, lens)
    n, seg = lo.vad_long(pcm, atap, max(int(n.max()), 1), lens)
    out = dict(atap=atap, n_segs=n, seg_off=np.zeros((B, max_segs, 2), np.uint32), frm_num=np.zeros((B, max_segs), np.uint32),
               seg_status=np.zeros((B, max_segs), np.uint8))
    seq_seg, seg_frm, dec = [0], [], []
    for b in range(B):
        for k in range(int(n[b])):
            st, en = int(seg[b, k, 0]), int(seg[b, k, 1])
            F = long_frames(st, en, U, 200 if geom_b else 160)
            ok = 1 <= F <= CONN_FRM_MAX
            seg_frm.append(F if ok else 0)
            if ok:
                dec.append((b, st, F))
            if k < max_segs:
                out["seg_off"][b, k] = st, en
                out["frm_num"][b, k] = F if ok else 0
                out["seg_status"][b, k] = 1 if en == NULL else 0 if ok else 2
        seq_seg.append(len(seg_frm))
    rows = [r for _, _, r in piece_features(port, pcm, atap, dec, geom_b)]
    feat = np.concatenate(rows).astype(np.int16) if rows else np.zeros((0, 12), np.int16)
    out["words"], out["n_words"], out["total"] = lg.decode_segs(feat, seq_seg, seg_frm, bank, n_slot, slot_stride, grammar,
                                                                penalty, max_words)
    return out


# ---- recordings and banks ---------------------------------------------------------------------------------------------
def golden_wav(name):
    """a digit recording of tests/golden as 12-bit ADC samples at 8 kHz"""
    import sr_b200
    with open(os.path.join(GOLDEN, name + ".wav"), "rb") as f:
        pcm, rate = sr_b200.wav_to_adc12(f.read())
    assert rate == 8000
    return pcm


def synth_bank(T=12, seed=0x7E3A0000):
    """T templates enrolled by the port from sr_synth_pcm_host: (bank, T)"""
    import sr_b200
    tpl = sr_b200.synth_pcm_host(T, 8000, seed)
    e = PortOracle().recognise_batch(tpl, 2400, None, 0, 4096)
    return sr_b200.make_bank(e["ftr"]), T


def synth_long(B, U, seed):
    """B synthetic recordings of U samples with many words: 2-second utterances of sr_synth_pcm_host (300 ms of noise,
    then 3 words) back to back, each shifted to the DC level of its recording's first one, so that VAD finds the words"""
    import sr_b200
    n = -(-U // 16000)
    utt = sr_b200.synth_pcm_host(B * n, 16000, seed, 3).reshape(B, n, 16000).astype(np.int32)
    dc = utt[:, :, :2400].mean(axis=2).round().astype(np.int32)
    utt += (dc[:, :1] - dc)[:, :, None]
    return np.ascontiguousarray(np.clip(utt, 0, 4095).astype(np.uint16).reshape(B, n * 16000)[:, :U])
