"""Closed-form tables (tools/gen_tables.py -> csrc/sr_tables.h) against the reference's own numbers (stored in
tests/golden/ref_tables.npz by tests/golden/make_golden.py), the
log threshold table against the host libm expression of MFCC.C:168, and the kernel's filter partition
against a brute-force restatement of MFCC.C:136-162. CPU only."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_tables  # noqa: E402
import oracle_bind as ob  # noqa: E402



def _ref_arrays():
    z = np.load(os.path.join(ROOT, "tests", "golden", "ref_tables.npz"))
    return {k: z[k].tolist() for k in z.files}


def test_mfcc_tables_equal_reference_header():
    r = _ref_arrays()
    cen, odd, even = gen_tables.tri_tables()
    assert gen_tables.hamm_table() == r["hamm"]           # MFCC_Arg.h:6-9
    assert cen == r["tri_cen"]                            # MFCC_Arg.h:12-15
    assert odd == r["tri_odd"]                            # MFCC_Arg.h:18-21
    assert even == r["tri_even"]                          # MFCC_Arg.h:24-27
    assert gen_tables.dct_table() == r["dct_arg"]         # MFCC_Arg.h:30-44


def test_twiddles_equal_reference_asm_table():
    vals = _ref_arrays()["twiddle"]
    assert len(vals) == 2040
    assert gen_tables.twiddle_table() == vals             # .s:285-629


def test_committed_header_is_current():
    """sr_tables.h in the tree is what the generator produces now, including the GEOM_B tables (kernel and oracle both read
    the header, so a stale one would pass every parity test)"""
    path = os.path.join(ROOT, "stm32-speech-recognition_b200", "csrc", "sr_tables.h")
    text = open(path).read()

    def table(name, n):
        return [int(x) for x in re.search(r"\b%s\[%d\] = \{([^}]*)\}" % (name, n), text).group(1).replace("\n", "").split(",")
                if x.strip()]
    assert table("sr_tab_hamm", 160) == gen_tables.hamm_table()
    assert table("sr_tab_twiddle", 2040) == gen_tables.twiddle_table()
    cen_b, odd_b, even_b = gen_tables.tri_tables(gen_tables.FRQ_MAX_B)
    assert table("sr_tab_b_hamm", 200) == gen_tables.hamm_table(gen_tables.FRAME_LEN_B)
    assert table("sr_tab_b_tri_cen", 24) == cen_b
    assert table("sr_tab_b_tri_odd", 128) == odd_b
    assert table("sr_tab_b_tri_even", 128) == even_b


def test_log_threshold_table_matches_libm_expression():
    """thr[L] is the first v with (u32)(log((double)v)*100) >= L for the host's libm (MFCC.C:168)"""
    thr, lmax = gen_tables.log_thresholds()
    assert lmax == 2218 and thr[0] == 1
    o = ob.port()
    for L in range(1, lmax + 1):
        v = thr[L]
        assert o.lib.sro_log100(v) >= L, (L, v)          # plateaus: thr[1..69] = 2 because log100(2) = 69
        assert o.lib.sro_log100(v - 1) < L, (L, v)
    assert o.lib.sro_log100(0) == 0 and o.lib.sro_log100(1) == 0 and o.lib.sro_log100(0xFFFFFFFF) == 2218
    # python's own double log agrees as well (same expression)
    rng = np.random.default_rng(3)
    for v in rng.integers(1, 2 ** 32, 2000, dtype=np.uint64).tolist():
        assert o.lib.sro_log100(v) == int(math.log(float(v)) * 100)


def test_filter_ranges_reproduce_reference_ranges():
    """the filter ranges and prefix-sum read positions used by mfcc_kernel are exactly the bins of MFCC.C:136-162"""
    import sr_b200
    L = sr_b200.lib()
    lo, hi, elo, ehi = (np.zeros(24, np.uint16) for _ in range(4))
    xlo, xhi = np.zeros(24, np.uint8), np.zeros(24, np.uint8)
    L.sr_debug_filter_ranges(*[a.ctypes.data_as(C.c_void_p) for a in (lo, hi, elo, ehi, xlo, xhi)])
    cen, _, _ = gen_tables.tri_tables()
    rng = {0: (0, cen[1]), 23: (cen[22], 512)}
    for h in range(2, 24, 2):
        rng[h] = (cen[h - 1], cen[h + 1])
    for h in range(1, 22, 2):
        rng[h] = (cen[h - 1], cen[h + 1])
    word = lambda l, i: 16 * l + 4 * ((i >> 2) ^ ((l >> 1) & 3)) + (i & 3)
    for h in range(24):
        assert (int(lo[h]), int(hi[h])) == rng[h], h
        for k, e, x in ((int(lo[h]), int(elo[h]), int(xlo[h])), (int(hi[h]), int(ehi[h]), int(xhi[h]))):
            assert x == k >> 4
            assert e == (1150 if k == 512 else (h & 1) * 512 + word(k >> 4, k & 15))
    # rows never overlap, stay inside the FFT scratch, and the 16-byte stores of 8 neighbouring lanes are conflict-free
    for q in range(4):
        for g in range(4):
            banks = set()
            for l in range(8 * q, 8 * q + 8):
                banks |= {(word(l, 4 * g) + c) % 32 for c in range(4)}
            assert len(banks) == 32
    used = set()
    for par in range(2):
        for l in range(32):
            for i in range(16):
                w = par * 512 + word(l, i)
                assert w not in used and w < 1084
                used.add(w)


def test_prefix_sum_filter_model_equals_direct_sums():
    """model of mfcc_kernel's filter stage (per-lane running totals + scanned lane totals, a filter = S(hi) - S(lo) read
    at the offsets of sr_debug_filter_ranges) against the direct sums of MFCC.C:136-162, all mod 2^32"""
    import sr_b200
    L = sr_b200.lib()
    lo, hi, elo, ehi = (np.zeros(24, np.uint16) for _ in range(4))
    xlo, xhi = np.zeros(24, np.uint8), np.zeros(24, np.uint8)
    L.sr_debug_filter_ranges(*[a.ctypes.data_as(C.c_void_p) for a in (lo, hi, elo, ehi, xlo, xhi)])
    cen, tri_odd, tri_even = gen_tables.tri_tables()
    tri = [np.array(tri_even, np.uint64), np.array(tri_odd, np.uint64)]
    rng = np.random.default_rng(11)
    word = lambda l, i: 16 * l + 4 * ((i >> 2) ^ ((l >> 1) & 3)) + (i & 3)
    M = np.uint64(0xFFFFFFFF)
    for trial in range(20):
        E = rng.integers(0, 2 ** 32, 512, dtype=np.uint64)
        if trial == 0:
            E[:] = 0xFFFFFFFF
        fb = np.zeros(1152, np.uint64)
        X = np.zeros((2, 33), np.uint64)
        TOT = [None, None]
        for par in range(2):
            v = ((E * tri[par]) & M) // np.uint64(100)
            tot = np.zeros(32, np.uint64)
            for l in range(32):
                run = np.uint64(0)
                for i in range(16):
                    fb[par * 512 + word(l, i)] = run
                    run = (run + v[16 * l + i]) & M
                tot[l] = run
            TOT[par] = tot
            inc = np.cumsum(tot) & M
            X[par, :32] = (inc - tot) & M
            X[par, 32] = inc[31]
        for h in range(24):
            par = h & 1
            got = ((X[par, xhi[h]] + fb[ehi[h]]) - (X[par, xlo[h]] + fb[elo[h]])) & M
            got2 = (fb[ehi[h]] - fb[elo[h]]) & M                       # the form without the scan: e_hi - e_lo + spanned lane totals
            assert int(xhi[h]) - int(xlo[h]) <= 6
            for l in range(int(xlo[h]), int(xhi[h])):
                got2 = (got2 + TOT[par][l]) & M
            assert got2 == got
            a, b = (0, cen[1]) if h == 0 else ((cen[22], 512) if h == 23 else (cen[h - 1], cen[h + 1]))
            want = np.uint64(0)
            for k in range(a, b):
                want = (want + ((E[k] * tri[par][k]) & M) // np.uint64(100)) & M
            assert got == want, (trial, h)
