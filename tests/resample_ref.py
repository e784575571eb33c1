"""numpy restatement of sr_resample_adc12_dev (include/sr_synth.h), the oracle of tests/test_resample.py.

(L, M) = (8000, rate) / gcd and h[0..N-1] is the rate's table (tools/gen_resample_taps.py, which the tests hold to the
committed header), centre c = (N-1)/2. With u[i] = x[i/L] - 2048 when i % L == 0 and 0 <= i/L < len, else 0:

  acc[n] = sum_k h[k] * u[n*M + c - k]            (exact in s32)
  y[n]   = clamp(2048 + ((acc[n] + 2^14) >> 15), 0, 4095)
  out_len = ceil(len * L / M), 0 when len = 0

Only the taps with n*M + c - k a multiple of L meet a sample, so output n reads phase p = (n*M + c) % L of the table,
h[p], h[p + L], ..., against x[j], x[j - 1], ... from j = (n*M + c) // L down."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_resample_taps as gen  # noqa: E402

RATES = gen.RATES


def ratio(rate):
    return gen.ratio(rate)


def taps(rate):
    return np.array(gen.taps(rate), np.int64)


def out_len(n, rate):
    L, M = ratio(rate)
    return 0 if n == 0 else -(-n * L // M)


def phases(rate):
    """the table as [L, K] phases, K = ceil(N / L), zero-padded: phase p holds h[p], h[p + L], ..."""
    h = taps(rate)
    L, _ = ratio(rate)
    K = -(-len(h) // L)
    hp = np.zeros(L * K, np.int64)
    hp[:len(h)] = h
    return hp.reshape(K, L).T.copy()


def accumulate(x, rate, idx):
    """acc[n] for the output indices idx (int64) of one recording x (its whole length is len)"""
    h = taps(rate)
    L, M = ratio(rate)
    c = (len(h) - 1) // 2
    hp = phases(rate)
    K = hp.shape[1]
    u = np.asarray(x, np.int64) - 2048
    t = np.asarray(idx, np.int64) * M + c
    ph, jhi = t % L, t // L
    # u with K - 1 zeros before it and enough after it for the last requested output
    hi = int(jhi.max()) + 1 if len(t) else 0
    upad = np.zeros(K - 1 + max(hi, len(u)), np.int64)
    upad[K - 1:K - 1 + len(u)] = u
    acc = np.zeros(len(t), np.int64)
    for m in range(K):
        acc += hp[ph, m] * upad[jhi - m + K - 1]
    assert (np.abs(acc) < 2 ** 31).all()
    return acc


def resample(x, rate, idx=None, chunk=1 << 16):
    """y (u16) of recording x at `rate`: all out_len outputs, or those at the indices idx"""
    x = np.asarray(x)
    if idx is None:
        idx = np.arange(out_len(len(x), rate), dtype=np.int64)
    idx = np.asarray(idx, np.int64)
    y = np.zeros(len(idx), np.uint16)
    for a in range(0, len(idx), chunk):
        acc = accumulate(x, rate, idx[a:a + chunk])
        y[a:a + chunk] = np.clip(2048 + ((acc + (1 << 14)) >> 15), 0, 4095)
    return y


def resample_batch(pcm, rate, lens, U_out, out=None):
    """[B, U_out] u16: row b holds resample(pcm[b, :lens[b]]) and keeps `out`'s bytes (zeros when None) past it"""
    B = pcm.shape[0]
    out = np.zeros((B, U_out), np.uint16) if out is None else out.copy()
    for b in range(B):
        y = resample(pcm[b, :int(lens[b])], rate)
        out[b, :len(y)] = y
    return out
