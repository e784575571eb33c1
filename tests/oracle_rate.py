"""Checker of the banded DP without the 2:1 length guard (SR_DTW_BAND | SR_DTW_ANY_RATE, include/speech_recog.h, TEST
INFRASTRUCTURE):
  RateOracle -- ctypes binding of oracle/_build/liboracle_rate.so, built by __graft_entry__.build() from tests/oracle_rate.c:
                the SR_DTW_BAND DP over every cell with the band test and no guard, scores of B inputs against a bank"""
import ctypes as C
import os

import numpy as np

from oracle_bind import FTR_DTYPE, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATE_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_rate.so")
UNREACHED = 2 ** 63 - 1


class RateOracle:
    name = "oracle-rate"

    def __init__(self):
        self.lib = C.CDLL(RATE_SO)
        self.lib.sro_rate_d.restype = C.c_int64
        self.lib.sro_rate_d.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]

    def d(self, x, y, r):
        """D(I-1, M-1) of rows x [I, 12] against y [M, 12] (1..119 rows each) at radius r, or None when unreachable"""
        x, y = np.ascontiguousarray(x, np.int16), np.ascontiguousarray(y, np.int16)
        v = self.lib.sro_rate_d(_p(x), len(x), _p(y), len(y), int(min(r, 118)))
        return None if v == UNREACHED else int(v)

    def dtw_batch(self, ftr_in, bank, n_slot, slot_stride, check_sign=0, band_r=0, nthreads=8):
        """score [B, n_slot] of FTR_DTYPE inputs against a bank of n_slot slots of slot_stride bytes"""
        ftr_in = np.ascontiguousarray(ftr_in, FTR_DTYPE)
        bank = np.ascontiguousarray(bank).view(np.uint8)
        B = ftr_in.shape[0]
        score = np.zeros((B, n_slot), np.uint32)
        if B and n_slot:
            self.lib.sro_rate_batch(_p(ftr_in), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
                                    C.c_int(check_sign), C.c_int(band_r), _p(score), C.c_int(nthreads))
        return score


def rate_oracle():
    return RateOracle()
