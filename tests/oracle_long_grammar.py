"""Checkers of the long-recording grammar decoder (include/sr_long_grammar.h, TEST INFRASTRUCTURE):
  LongGrammarOracle       -- ctypes binding of oracle/_build/liboracle_long_grammar.so, built by __graft_entry__.build()
                             from tests/oracle_long_grammar.c: the CPU restatement of sr_connected_grammar_segs_batch
  recognise_long_grammar  -- sr_recognise_long_grammar_batch composed from the long-form VAD oracle, the port's
                             noise_atap and piece-wise get_mfcc, and that restatement"""
import ctypes as C
import os

import numpy as np

from oracle_bind import NULL, _p
from oracle_connected import CONN_FRM_MAX, WORD_DTYPE, long_frames
from oracle_grammar import _arcs
from oracle_long import atap_long

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LONG_GRAMMAR_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_long_grammar.so")
LONG_GRAM_FRM_MAX = 1677720


class LongGrammarOracle:
    name = "oracle-long-grammar"

    def __init__(self):
        self.lib = C.CDLL(LONG_GRAMMAR_SO)

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
        bank = np.ascontiguousarray(bank, np.uint8) if n_slot else np.zeros(16, np.uint8)
        S, F, n_arcs, arcs = _arcs(grammar)
        words = np.zeros((B, max_words), WORD_DTYPE)
        n_words, total = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
        self.lib.sro_long_grammar_batch(_p(feat), _p(seq_seg), _p(seg_frm), C.c_uint32(B), _p(bank), C.c_uint32(n_slot),
                                        C.c_uint32(slot_stride), C.c_uint32(S), C.c_uint32(F), C.c_uint32(n_arcs), _p(arcs),
                                        C.c_uint32(penalty), C.c_uint32(max_words), _p(words), _p(n_words), _p(total),
                                        C.c_int(nthreads))
        return words, n_words, total


def long_grammar():
    return LongGrammarOracle()


def segment_features(port, pcm, atap, segs, geom_b=False):
    """sr_mfcc_long_batch's features of (b, start, end, F) segments from the port's get_mfcc, piece by piece: piece k of a
    segment starts at sample start + 80*119*k and reads its real preceding sample (mid_val at sample 0). Returns the
    segments' rows back to back, [sum F, 12] i16"""
    frame_len = 200 if geom_b else 160
    pieces = []
    for b, st, _, F in segs:
        for f0 in range(0, F, 119):
            nf = min(119, F - f0)
            ps = st + 80 * f0
            pieces.append((b, nf, ps, ps + 80 * (nf - 1) + frame_len))
    if not pieces:
        return np.zeros((0, 12), np.int16)
    L = max(pe - ps for _, _, ps, pe in pieces)
    xs = np.zeros((len(pieces), L + 1), np.uint16)           # [x[-1], samples]
    for i, (b, _, ps, pe) in enumerate(pieces):
        xs[i, 0] = pcm[b, ps - 1] if ps else np.uint16(atap["mid_val"][b] & 0xFFFF)
        xs[i, 1:1 + pe - ps] = pcm[b, ps:pe]
    s2 = np.array([[1, 1 + pe - ps] for _, _, ps, pe in pieces], np.uint32)
    at = atap[[p[0] for p in pieces]]
    f = port.mfcc_geom_b_batch(xs, s2, at) if geom_b else port.mfcc_batch(xs, s2, at, nthreads=8)
    out = []
    for q, (_, nf, _, _) in enumerate(pieces):
        assert int(f["frm_num"][q]) == nf
        out.append(f["mfcc_dat"][q][: nf * 12].reshape(nf, 12))
    return np.concatenate(out).astype(np.int16)


def recognise_long_grammar(lo, port, lg, pcm, n_len, bank, n_slot, slot_stride, grammar, penalty, max_segs, max_words,
                           lens=None, geom_b=False, atap=None):
    """sr_recognise_long_grammar_batch from the oracles' stages: the long-form VAD of every segment, each decodable one's
    features, one decode per recording over its flat segment table. Returns a dict of the sr_long_gram_out fields (records
    past n_segs / n_words zero)"""
    B, U = pcm.shape
    atap = atap_long(port, pcm, n_len, lens, atap)
    n, _ = lo.vad_long(pcm, atap, 0, lens)
    n, seg = lo.vad_long(pcm, atap, max(int(n.max()), 1), lens)
    frame_len = 200 if geom_b else 160
    out = dict(atap=atap, n_segs=n, seg_off=np.zeros((B, max_segs, 2), np.uint32), frm_num=np.zeros((B, max_segs), np.uint32),
               seg_status=np.zeros((B, max_segs), np.uint8))
    seq_seg, seg_frm, dec = [0], [], []
    for b in range(B):
        for k in range(int(n[b])):
            st, en = int(seg[b, k, 0]), int(seg[b, k, 1])
            F = long_frames(st, en, U, frame_len)
            ok = 1 <= F <= CONN_FRM_MAX
            seg_frm.append(F if ok else 0)
            if ok:
                dec.append((b, st, en, F))
            if k < max_segs:
                out["seg_off"][b, k] = st, en
                out["frm_num"][b, k] = F if ok else 0
                out["seg_status"][b, k] = 1 if en == NULL else 0 if ok else 2
        seq_seg.append(len(seg_frm))
    feat = segment_features(port, pcm, atap, dec, geom_b)
    out["words"], out["n_words"], out["total"] = lg.decode_segs(feat, seq_seg, seg_frm, bank, n_slot, slot_stride, grammar,
                                                                penalty, max_words)
    return out
