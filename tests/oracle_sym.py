"""Checker of the symmetric slope-constrained matcher (SR_DTW_SYM_P1, include/speech_recog.h, TEST INFRASTRUCTURE):
  SymOracle -- ctypes binding of oracle/_build/liboracle_sym.so, built by __graft_entry__.build() from tests/oracle_sym.c:
               Sakoe & Chiba's symmetric P = 1 DP over SR_DTW_BAND's band, scores of B inputs against a bank"""
import ctypes as C
import os

import numpy as np

from oracle_bind import FTR_DTYPE, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYM_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_sym.so")
UNREACHED = 2 ** 64 - 1


class SymOracle:
    name = "oracle-sym"

    def __init__(self):
        self.lib = C.CDLL(SYM_SO)
        self.lib.sro_sym_get_dis.restype = C.c_uint32
        self.lib.sro_sym_g.restype = C.c_uint64
        self.lib.sro_sym_g.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
        self.lib.sro_sym.restype = C.c_uint32

    def g(self, x, y, r):
        """g(I-1, M-1) of rows x [I, 12] against y [M, 12] (1..119 rows each) at radius r, or None when unreachable"""
        x, y = np.ascontiguousarray(x, np.int16), np.ascontiguousarray(y, np.int16)
        v = self.lib.sro_sym_g(_p(x), len(x), _p(y), len(y), int(min(r, 118)))
        return None if v == UNREACHED else int(v)

    def dtw_batch(self, ftr_in, bank, n_slot, slot_stride, check_sign=0, band_r=0, nthreads=8):
        """score [B, n_slot] of FTR_DTYPE inputs against a bank of n_slot slots of slot_stride bytes"""
        ftr_in = np.ascontiguousarray(ftr_in, FTR_DTYPE)
        bank = np.ascontiguousarray(bank).view(np.uint8)
        B = ftr_in.shape[0]
        score = np.zeros((B, n_slot), np.uint32)
        if B and n_slot:
            self.lib.sro_sym_batch(_p(ftr_in), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
                                   C.c_int(check_sign), C.c_int(band_r), _p(score), C.c_int(nthreads))
        return score


def sym_oracle():
    return SymOracle()
