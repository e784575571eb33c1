"""Checkers of the grammar decoder (TEST INFRASTRUCTURE):
  GrammarOracle  -- ctypes binding of oracle/_build/liboracle_grammar.so, built by __graft_entry__.build() from
                    tests/oracle_grammar.c: the CPU restatement of sr_connected_grammar_batch, with segments
  recognise_connected_grammar -- sr_recognise_connected_grammar_batch composed from the oracle stages"""
import ctypes as C
import os

import numpy as np

from oracle_bind import ATAP_DTYPE, NULL, _p
from oracle_connected import CONN_FRM_MAX, WORD_DTYPE, mfcc_long

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAMMAR_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_grammar.so")
SEG_NONE = 0xFFFFFFFF


def _arcs(g):
    n_states, final_mask, arcs = g
    a = np.array(arcs, np.uint32).reshape(-1, 3) if arcs else np.zeros((1, 3), np.uint32)
    return int(n_states), int(final_mask), len(arcs), np.ascontiguousarray(a)


class GrammarOracle:
    name = "oracle-grammar"

    def __init__(self):
        self.lib = C.CDLL(GRAMMAR_SO)

    def decode(self, feat, frm, bank, n_slot, slot_stride, grammar, penalty, max_words, seg=None, nthreads=1):
        """feat [B, stride, 12] i16, frm [B], grammar (n_states, final_mask, [(from, to, cmd_mask), ...]), seg [B, 3]
        segment first frames (SEG_NONE: no frames) or None -> (words [B, max_words] WORD_DTYPE (zeros past n_words),
        n_words [B], total [B] u64)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm = np.ascontiguousarray(frm, np.uint32)
        bank = np.ascontiguousarray(bank, np.uint8) if n_slot else np.zeros(16, np.uint8)
        S, F, n_arcs, arcs = _arcs(grammar)
        seg = None if seg is None else np.ascontiguousarray(seg, np.uint32).reshape(B, 3)
        words = np.zeros((B, max_words), WORD_DTYPE)
        n_words, total = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
        self.lib.sro_grammar_batch(_p(feat), _p(frm), C.c_uint32(stride), _p(seg), C.c_uint32(B), _p(bank),
                                   C.c_uint32(n_slot), C.c_uint32(slot_stride), C.c_uint32(S), C.c_uint32(F),
                                   C.c_uint32(n_arcs), _p(arcs), C.c_uint32(penalty), C.c_uint32(max_words), _p(words),
                                   _p(n_words), _p(total), C.c_int(nthreads))
        return words, n_words, total


def grammar():
    return GrammarOracle()


def recognise_connected_grammar(ora, go, pcm, n_len, bank, n_slot, slot_stride, grammar_, penalty, max_words, geom_b=False,
                                atap0=None, nthreads=1):
    """sr_recognise_connected_grammar_batch composed from the oracle stages: noise_atap and VAD per row, mfcc_long of every
    segment at frm_cap = 818, each capture's segments with frames back to back as one sequence decoded under the grammar
    with its segment table, status from segment 0. Returns a dict of the sr_conn_out fields (words zero past n_words)"""
    B, U = pcm.shape
    out = dict(atap=np.zeros(B, ATAP_DTYPE), seg_off=np.zeros((B, 3, 2), np.uint32), frm_num=np.zeros((B, 3), np.uint32),
               status=np.zeros(B, np.uint8))
    for b in range(B):
        out["atap"][b] = ora.noise_atap(pcm[b], n_len, None if atap0 is None else atap0[b:b + 1])[0]
        out["seg_off"][b] = ora.vad(pcm[b], U, out["atap"][b:b + 1]).reshape(3, 2)
    feats = []
    for k in range(3):
        f, n = mfcc_long(ora, pcm, out["seg_off"][:, k, :], out["atap"], CONN_FRM_MAX, geom_b)
        feats.append(f)
        out["frm_num"][:, k] = n
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
        out["status"][b] = 1 if out["seg_off"][b, 0, 1] == NULL else 2 if out["frm_num"][b, 0] == 0 else 0
    out["words"], out["n_words"], out["total"] = go.decode(x, N, bank, n_slot, slot_stride, grammar_, penalty, max_words,
                                                           seg=seg, nthreads=nthreads)
    return out
