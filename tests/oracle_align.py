"""ctypes binding of the alignment oracle (TEST INFRASTRUCTURE): oracle/_build/liboracle_align.so, built by
__graft_entry__.build() from tests/oracle_align.c -- the CPU restatement of sr_dtw_path_batch and sr_average_bank."""
import ctypes as C
import os

import numpy as np

from oracle_bind import FTR_DTYPE, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALIGN_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_align.so")
PATH_MAX = 237


class AlignOracle:
    name = "oracle-align"

    def __init__(self):
        self.lib = C.CDLL(ALIGN_SO)
        self.lib.sro_dtw_path.restype = C.c_uint32

    def dtw_path(self, fin, fmdl, r, nthreads=1, with_path=True):
        """n pairs (fin[p], fmdl[p]) -> (dis [n], path [n, 237, 2] or None, path_len [n] or None)"""
        fin, fmdl = np.ascontiguousarray(fin, FTR_DTYPE), np.ascontiguousarray(fmdl, FTR_DTYPE)
        n = len(fin)
        assert len(fmdl) == n
        dis = np.zeros(n, np.uint32)
        path = np.zeros((n, PATH_MAX, 2), np.uint8) if with_path else None
        plen = np.zeros(n, np.uint32) if with_path else None
        self.lib.sro_dtw_path_batch(_p(fin), _p(fmdl), C.c_uint32(n), C.c_int(min(r, 2 ** 31 - 1)), _p(path), _p(plen),
                                    _p(dis), C.c_int(nthreads))
        return dis, path, plen

    def average_bank(self, bank, slot_stride, K, r, iters, nthreads=1):
        """bank [G*K, slot_stride] u8 -> (bank_out of the same shape, score [G, K], anchor [G])"""
        bank = np.ascontiguousarray(bank, np.uint8).reshape(-1, slot_stride)
        G = bank.shape[0] // K
        out = np.zeros_like(bank)
        score, anchor = np.zeros((G, K), np.uint32), np.zeros(G, np.uint32)
        self.lib.sro_average_bank(_p(bank), C.c_uint32(slot_stride), C.c_uint32(K), C.c_uint32(G), C.c_int(r),
                                  C.c_uint32(iters), _p(out), _p(score), _p(anchor), C.c_int(nthreads))
        return out, score, anchor


def align():
    return AlignOracle()
