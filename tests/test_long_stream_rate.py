"""Live streams at any rate of SR_RESAMPLE_RATES (sr_long_streams_create_at_rate, include/sr_synth.h; K14 at a rate in
csrc/sr_long_stream.cu): every push resamples each stream's chunk to 8 kHz on the GPU, carrying the filter's history
across pushes, before the long-form VAD and recognition of the 8 kHz pool.

The definition: after n_in input samples a stream's 8 kHz stream is the first n8(n_in) = max(0, ceil((n_in L - c) / M))
outputs of sr_resample_adc12_dev on them, and every rule of include/sr_long_stream.h holds on it. So every GPU test here
compares the pool, after every push or every few, with sr_resample_adc12_dev on the n_in samples followed by
sr_recognise_long_batch on the first n8 outputs (both pinned to their oracles elsewhere), and a few with the CPU
composition tests/resample_ref.py + the long-form oracle.

CPU: n8 as a property of the restatement (its first n8(n) outputs never change when input is added) and of the indices
(output n8(n) is the first whose support reaches input n), the max8 bound, and the header and the binding.
GPU: chunk lengths 1, M - 1, M, M + 1, 10 ms, 80 ms and max_chunk at every rate; random ragged pushes with zeros and a
late start; single-sample pushes, most of which complete no 8 kHz sample; rate 8000 against the plain pool; the digit
recordings at 16, 44.1 and 48 kHz; one push of 2^20 samples from pinned memory; subset resets; matchers and banks
switched between pushes; the launch count; refusals; the 2^32 - 1 input limit; the bytes a push reads and writes; two
handles on two threads. include/sr_synth.h is not enumerated by tests/test_concurrency.py, so the threaded check is
here."""
import ctypes as C
import inspect
import os
import re
import threading

import numpy as np
import pytest
from scipy.signal import resample_poly

import oracle_bind as ob
import oracle_ext as ox
import resample_ref as rr
import sr_b200
from cases import DIGITS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = 0xFFFFFFFF
ST_VAD_FAIL = 1
REC = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")
HEADER = open(os.path.join(ROOT, "include", "sr_long_stream.h")).read()
HISTORY = int(re.search(r"#define SR_LONG_STREAM_HISTORY\s+(\d+)u", HEADER).group(1))
POISON = 0xFFFF                    # past lens[s] in every chunk: a sample read from there would change the outputs


# ---- the definition, restated ---------------------------------------------------------------------------------------------
def geom(rate):
    L, M = rr.ratio(rate)
    N = len(rr.taps(rate))
    return L, M, (N - 1) // 2, -(-N // L)


def n8(n, rate):
    L, M, c, _ = geom(rate)
    return max(0, -(-(n * L - c) // M))


def max8(max_chunk, rate):
    L, M, _, _ = geom(rate)
    return -(-max_chunk * L // M)


def ring_len(max_chunk, n_len, rate):
    return -(-(max(n_len, HISTORY) + max8(max_chunk, rate)) // 80) * 80


def max_events(S, max_chunk, n_len, rate):
    c = n_len if n_len and n_len % 240 == 0 else 0
    return S * -(-(-(-(max8(max_chunk, rate) + c) // 80)) // 19)


def at_rate(x, rate):
    """8 kHz codes -> codes at `rate` (scipy's polyphase filter), rounded and clipped to 12 bits"""
    L, M = rr.ratio(rate)
    y = resample_poly(np.asarray(x, np.float64) - 2048, M, L)
    return np.clip(np.rint(y + 2048), 0, 4095).astype(np.uint16)


# ---- CPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", rr.RATES)
def test_first_n8_outputs_never_change(rate):
    """resample_ref on every prefix, and on random continuations of it, keeps the first n8(n) outputs of the whole"""
    rng = np.random.default_rng(rate + 1)
    L, M, c, K = geom(rate)
    top = 1000 if L > 1 else 2000
    x = rng.integers(0, 4096, top).astype(np.uint16)
    full = rr.resample(x, rate)
    for n in range(top + 1):
        k = n8(n, rate)
        assert k <= rr.out_len(n, rate)
        got = rr.resample(x[:n], rate, np.arange(k)) if k else full[:0]
        assert np.array_equal(got, full[:k]), (rate, n)
    for n in rng.integers(0, top, 20):
        tail = rng.integers(0, 4096, int(rng.integers(1, 3 * K))).astype(np.uint16)
        k = n8(int(n), rate)
        y = rr.resample(np.concatenate([x[:n], tail]), rate, np.arange(k))
        assert np.array_equal(y, full[:k]), (rate, n)


@pytest.mark.parametrize("rate", rr.RATES)
def test_output_n8_is_the_first_whose_support_reaches_input_n(rate):
    """a statement about indices: output k reads inputs (kM + c) // L - K + 1 .. (kM + c) // L"""
    L, M, c, K = geom(rate)
    n = np.arange(0, 200000, dtype=np.int64)
    k = np.maximum(0, -(-(n * L - c) // M))
    assert ((k * M + c) // L >= n).all()                                   # output n8(n) reads input n or later
    prev = k[k > 0] - 1
    assert ((prev * M + c) // L < n[k > 0]).all()                          # the one before it reads only inputs < n
    assert all(n8(int(v), rate) == int(w) for v, w in zip(n[::997], k[::997]))


@pytest.mark.parametrize("rate", rr.RATES)
def test_one_push_completes_at_most_max8_samples(rate):
    L, M, c, _ = geom(rate)
    n = np.arange(0, 20000, dtype=np.int64)
    f = lambda v: np.maximum(0, -(-(v * L - c) // M))                      # noqa: E731
    for b in (0, 1, M - 1, M, M + 1, 441, 480, 3528, 4410, 4800, 7777):
        d = f(n + b) - f(n)
        bound = -(-b * L // M)
        assert (d <= bound).all() and (d == bound).any(), (rate, b)


def test_header_and_binding():
    text = open(os.path.join(ROOT, "include", "sr_synth.h")).read()
    decl = re.search(r"int sr_long_streams_create_at_rate\(([^;]*)\);", text)
    assert decl and decl.group(1).count(",") == 6
    assert "max8 = ceil(max_chunk*L/M)" in text and "n8(n_in) = max(0, ceil((n_in*L - c) / M))" in text
    assert '#include "sr_long_stream.h"' in text
    # sr_long_stream.h keeps its own ten calls; the call at a rate is sr_synth.h's
    assert "sr_long_streams_create_at_rate" not in HEADER
    assert hasattr(sr_b200.lib(), "sr_long_streams_create_at_rate")
    sig = inspect.signature(sr_b200.LongStreamPool.__init__)
    assert sig.parameters["rate"].default is None
    assert max8(1, 44100) == 1 and max8(441, 44100) == 80 and max8(442, 44100) == 81 and max8(1 << 20, 8000) == 1 << 20
    assert ring_len(480, 2400, 48000) == ring_len(80, 2400, 8000) == -(-(HISTORY + 80) // 80) * 80
    assert max_events(10, 4800, 2400, 48000) == max_events(10, 800, 2400, 8000)


# ---- the reference: sr_resample_adc12_dev, then sr_recognise_long_batch ------------------------------------------------------
def gpu_eight(xs, ns, rate):
    """sr_resample_adc12_dev on xs[s][:ns[s]] for every stream, cut to the first n8(ns[s]) outputs"""
    import torch
    S = len(xs)
    U = max(1, max(int(n) for n in ns))
    pcm = np.zeros((S, U), np.uint16)
    for s in range(S):
        pcm[s, :ns[s]] = xs[s][:ns[s]]
    U_out = rr.out_len(U, rate)
    x = torch.from_numpy(pcm.view(np.int16)).to("cuda:0")
    ln = torch.from_numpy(np.asarray(ns, np.uint32).view(np.int32)).to("cuda:0")
    out = torch.zeros((S, max(U_out, 1)), dtype=torch.int16, device="cuda:0")
    s0 = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U, S, ln.data_ptr(), rate, out.data_ptr(), U_out, None, s0.cuda_stream)
    s0.synchronize()
    y = out.cpu().numpy().view(np.uint16)
    return [y[s, :n8(int(ns[s]), rate)].copy() for s in range(S)]


def expected(h, eights, n_len, atap0, rows):
    """sr_recognise_long_batch on each 8 kHz prefix: per stream (closed records, open start, atap)"""
    U = max(1, max(len(eights[s]) for s in rows))
    pcm = np.zeros((len(rows), U), np.uint16)
    lens = np.zeros(len(rows), np.uint32)
    for i, s in enumerate(rows):
        pcm[i, :len(eights[s])] = eights[s]
        lens[i] = len(eights[s])
    atap = np.zeros(len(rows), sr_b200.ATAP_DTYPE) if atap0 is None else np.ascontiguousarray(atap0[rows])
    max_segs = int(lens.max()) // (19 * 80) + 4
    r = h.recognise_long_batch(pcm, max_segs, n_len, lens, atap)
    out = {}
    for i, s in enumerate(rows):
        recs = [tuple(int(v) for v in rec) for rec in r["segs"][i, :int(r["n_segs"][i])].tolist()]
        closed = [t for t in recs if t[2] != ST_VAD_FAIL]
        op = recs[-1][0] if recs and recs[-1][2] == ST_VAD_FAIL else NULL
        out[s] = (closed, op, r["atap"][i].tobytes())
    return out


class Feed:
    """a pool at `rate` and its streams: ragged pushes with poison past every length, each stream's events in order, and
    the check against K15 + sr_recognise_long_batch on the same input"""

    def __init__(self, h, xs, max_chunk, rate, n_len=2400, atap0=None, pool_rate="same"):
        self.h, self.xs, self.rate, self.n_len, self.atap0 = h, [np.asarray(x, np.uint16) for x in xs], rate, n_len, atap0
        self.S = len(xs)
        self.pool = sr_b200.LongStreamPool(h, self.S, max_chunk, n_len, atap0, rate=rate if pool_rate == "same" else pool_rate)
        self.n = np.zeros(self.S, np.int64)
        self.got = [[] for _ in range(self.S)]

    def take(self, evs):
        for e in evs:
            assert e["segment"] == len(self.got[e["stream"]]), e
            self.got[e["stream"]].append(tuple(int(e[k]) for k in REC))

    def chunk(self, lens):
        lens = np.asarray(lens, np.int64)
        chunk = np.full((self.S, max(1, int(lens.max()))), POISON, np.uint16)
        for s in range(self.S):
            chunk[s, :lens[s]] = self.xs[s][self.n[s]:self.n[s] + lens[s]]
            assert (chunk[s, :lens[s]] < 4096).all() and self.n[s] + lens[s] <= len(self.xs[s])
        return chunk

    def push(self, lens):
        lens = np.asarray(lens, np.int64)
        self.take(self.pool.push_ragged(self.chunk(lens), lens.astype(np.uint32)))
        self.n += lens

    def check(self, rows=None):
        st = self.pool.state()
        assert [int(v) for v in st["n_recv"]] == [n8(int(n), self.rate) for n in self.n]
        eights = gpu_eight(self.xs, self.n, self.rate)
        rows = [s for s in (range(self.S) if rows is None else rows)
                if len(eights[s]) > 0 and (len(eights[s]) >= self.n_len or not (self.n_len and self.n_len % 240 == 0))]
        if not rows:
            return
        want = expected(self.h, eights, self.n_len, self.atap0, rows)
        for s in rows:
            closed, op, atap = want[s]
            assert self.got[s] == closed, (s, int(self.n[s]), self.got[s][-3:], closed[-3:])
            assert int(st["n_closed"][s]) == len(closed)
            assert int(st["open_start"][s]) == op, (s, int(self.n[s]))
            assert st["atap"][s].tobytes() == atap, s

    def check_cpu(self, s, bank):
        """stream s against the CPU composition: resample_ref, then the long-form oracle"""
        y = rr.resample(self.xs[s][:self.n[s]], self.rate, np.arange(n8(int(self.n[s]), self.rate)))
        lo, port = ox.long_oracle(), ob.port()
        max_segs = len(y) // (19 * 80) + 4
        r = ox.recognise_long(lo, port, y[None], self.n_len, bank[0], bank[1], 4096, max_segs)
        recs = [tuple(int(rec[k]) for k in REC) for rec in r["segs"][0, :int(r["n_segs"][0])]]
        assert self.got[s] == [t for t in recs if t[2] != ST_VAD_FAIL]

    def close(self):
        self.pool.close()


def _uniform(total, c):
    out, n = [], 0
    while n < total:
        out.append(min(c, total - n))
        n += out[-1]
    return out


def _schedule(total, pattern):
    """pushes cycling through `pattern` until `total` samples are in"""
    out, n, i = [], 0, 0
    while n < total:
        out.append(min(pattern[i % len(pattern)], total - n))
        n += out[-1]
        i += 1
    return out


def _drive(feed, per_stream, every=1):
    """per_stream[s]: stream s's pushes; stream s pushes 0 once its list is done"""
    steps = max(len(p) for p in per_stream)
    for i in range(steps):
        feed.push([p[i] if i < len(p) else 0 for p in per_stream])
        if every and (i % every == 0 or i == steps - 1):
            feed.check()


def synth_at(rate, S, n8k, seed):
    return [at_rate(x, rate) for x in ox.synth_long(S, n8k, seed)]


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bank():
    return ox.synth_bank()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", rr.RATES)
def test_chunk_lengths(handle, bank, rate):
    """stream 0 cycles 1, M - 1, M, M + 1, 10 ms and 80 ms; streams 1-3 push 10 ms, 80 ms and max_chunk at a time"""
    handle.set_bank(bank[0], bank[1], 4096)
    L, M, _, _ = geom(rate)
    ms10, ms80, max_chunk = rate // 100, rate // 100 * 8, rate // 10 + 7
    xs = synth_at(rate, 4, 24000, 0x15A0 + rate)
    N = len(xs[0])
    f = Feed(handle, xs, max_chunk, rate)
    assert f.pool.ring_len == ring_len(max_chunk, 2400, rate) and f.pool.max_events == max_events(4, max_chunk, 2400, rate)
    _drive(f, [_schedule(N, [1, M - 1, M, M + 1, ms10, ms80]), _uniform(N, ms10), _uniform(N, ms80),
               _uniform(N, max_chunk)], every=3)
    assert sum(len(g) for g in f.got) > 4
    f.check_cpu(1, bank)
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [11025, 44100, 48000])
def test_random_ragged_pushes(handle, bank, rate):
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(rate)
    S, max_chunk = 6, rate // 12
    xs = synth_at(rate, S, 32000, 0x15B0)
    N = len(xs[0])
    f = Feed(handle, xs, max_chunk, rate)
    start = np.zeros(S, int)
    start[2] = 15                                       # a stream that starts late
    i = 0
    while (f.n < N).any():
        lens = rng.integers(0, max_chunk + 1, S)
        lens[rng.random(S) < 0.2] = 0
        lens[i < start] = 0
        f.push(np.minimum(lens, N - f.n))
        f.check()
        i += 1
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", rr.RATES)
def test_single_samples_and_pushes_that_complete_nothing(handle, rate):
    """n_recv follows n8 sample by sample through the first ceil((c + 1) / L) inputs, which complete no 8 kHz sample,
    and through zero-length pushes"""
    L, M, c, K = geom(rate)
    xs = [np.full(4 * K * M // L + 400, 2048 + 7 * s, np.uint16) for s in range(2)]
    f = Feed(handle, xs, 64, rate)
    silent = 0
    for i in range(len(xs[0])):
        before = f.pool.state()["n_recv"].copy()
        f.push([1, i % 2])
        st = f.pool.state()
        assert [int(v) for v in st["n_recv"]] == [n8(int(n), rate) for n in f.n], i
        silent += int((st["n_recv"] == before).all())
    assert silent > 0 or rate == 8000
    f.check()
    f.close()


@pytest.mark.gpu
def test_8000_is_the_plain_pool(handle, bank):
    """rate 8000: the same ring, events, state and launches as sr_long_streams_create, push for push"""
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(8)
    S, N, max_chunk = 5, 30000, 900
    xs = ox.synth_long(S, N, 0x15C0)
    a = Feed(handle, list(xs), max_chunk, 8000)
    b = Feed(handle, list(xs), max_chunk, 8000, pool_rate=None)
    assert (a.pool.ring_len, a.pool.max_events) == (b.pool.ring_len, b.pool.max_events)
    while (a.n < N).any():
        lens = np.minimum(rng.integers(0, max_chunk + 1, S), N - a.n)
        chunk = a.chunk(lens)
        l0 = handle.launch_count()
        ea = a.pool.push_ragged(chunk, lens.astype(np.uint32))
        l1 = handle.launch_count()
        eb = b.pool.push_ragged(chunk, lens.astype(np.uint32))
        assert l1 - l0 == handle.launch_count() - l1
        assert ea == eb
        a.take(ea)
        a.n += lens
        sa, sb = a.pool.state(), b.pool.state()
        assert all(sa[k].tobytes() == sb[k].tobytes() for k in sa)
    a.check()
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_digit_recordings(handle, rate):
    lo, port = ox.long_oracle(), ob.port()
    from cases import digit_bank
    bk, T, _ = digit_bank(port, lo, ox.golden_wav(DIGITS[1]))
    handle.set_bank(bk, T, 4096)
    xs = [at_rate(ox.golden_wav(n), rate) for n in DIGITS]
    f = Feed(handle, xs, rate // 100, rate)
    N = np.array([len(x) for x in xs])
    i = 0
    while (f.n < N).any():
        f.push(np.minimum(rate // 100, N - f.n))
        if i % 25 == 0:
            f.check()
        i += 1
    f.check()
    assert sum(len(g) for g in f.got) > 10, [len(g) for g in f.got]
    f.check_cpu(0, (bk, T))
    f.close()


@pytest.mark.gpu
def test_one_push_of_2_20_samples_at_48k_from_pinned_memory(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    rate, S, big = 48000, 2, 1 << 20
    xs = synth_at(rate, S, (big + 5000) // 6 + 10, 0x15D0)
    f = Feed(handle, xs, big, rate)
    mem, ptr = sr_b200.host_alloc_dev(0, S * big * 2)
    buf = mem.view(np.uint16).reshape(S, big)
    try:
        for lens in ([big, 4321], [3000, big]):
            lens = np.minimum(lens, [len(x) for x in xs] - f.n)
            buf[:] = POISON
            for s in range(S):
                buf[s, :lens[s]] = xs[s][f.n[s]:f.n[s] + lens[s]]
            f.take(f.pool.push_ragged(ptr, np.asarray(lens, np.uint32), stride=big))
            f.n += lens
            f.check()
        assert len(f.got[0]) >= 10
    finally:
        f.close()
        sr_b200.host_free(ptr)


@pytest.mark.gpu
def test_reset_a_subset_mid_stream(handle, bank):
    """a reset stream equals a fresh pool fed what follows; the others carry on"""
    handle.set_bank(bank[0], bank[1], 4096)
    rate, S = 44100, 5
    c = rate // 100 + 13
    xs = synth_at(rate, S, 40000, 0x15E0)
    N = len(xs[0])
    f = Feed(handle, xs, c, rate)
    for k in _uniform(N // 2 + 321, c):
        f.push([k] * S)
    which = np.zeros(S, np.uint8)
    which[[1, 3]] = 1
    f.pool.reset(which)
    cut = int(f.n[1])
    fresh = Feed(handle, [f.xs[s][cut:] for s in (1, 3)], c, rate)
    for s in (1, 3):
        f.xs[s] = f.xs[s][cut:].copy()
        f.n[s] = 0
        f.got[s] = []
    while (f.n[[0, 2, 4]] < N).any():
        lens = np.minimum(c, np.array([len(x) for x in f.xs]) - f.n)
        f.push(lens)
        fresh.push(lens[[1, 3]])
    f.check()
    fresh.check()
    assert [f.got[1], f.got[3]] == fresh.got and len(f.got[1]) > 2
    f.close()
    fresh.close()


@pytest.mark.gpu
def test_matchers_and_bank_switched_between_pushes(handle, bank):
    bank2 = ox.synth_bank(9, 0x7E3B0000)
    rate, S = 48000, 4
    c = rate // 100 * 8
    xs = synth_at(rate, S, 48000, 0x15F0)
    configs = [(0, 0, bank), (sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE | sr_b200.dtw_reject(30), 118, bank2),
               (sr_b200.dtw_reject(80), 0, bank2), (sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE, 118, bank)]
    f = Feed(handle, xs, c, rate)
    rng = np.random.default_rng(3)
    try:
        for i, k in enumerate(_uniform(len(xs[0]), c)):
            flags, r, b = configs[int(rng.integers(len(configs)))]
            handle.set_match(flags, r)
            handle.set_bank(b[0], b[1], 4096)
            before = [len(g) for g in f.got]
            f.push([k] * S)
            if any(len(g) > n0 for g, n0 in zip(f.got, before)):
                want = expected(handle, gpu_eight(f.xs, f.n, rate), 2400, None, list(range(S)))
                for s in range(S):
                    assert f.got[s][before[s]:] == want[s][0][before[s]:len(f.got[s])], (i, s)
        assert sum(len(g) for g in f.got) > 10
    finally:
        handle.set_match(0, 0)
    f.close()


@pytest.mark.gpu
def test_launches_per_push(handle, bank):
    rate, S = 44100, 16
    c = rate // 100
    xs = np.array(synth_at(rate, S, 8000, 0x1600))
    pool = sr_b200.LongStreamPool(handle, S, c, 2400, rate=rate)
    try:
        for with_bank in (True, False):
            handle.set_bank(*((bank[0], bank[1]) if with_bank else (np.zeros((0, 4096), np.uint8), 0)), 4096)
            pool.reset()
            for i in range(0, xs.shape[1] - c, c):
                before = handle.launch_count()
                pool.push(np.ascontiguousarray(xs[:, i:i + c]))
                assert handle.launch_count() - before == (6 if with_bank else 5)
    finally:
        pool.close()


@pytest.mark.gpu
def test_refusals_write_nothing(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    for rate, mc in ((0, 480), (7999, 480), (12000, 480), (96000, 480), (44100, 0), (48000, (1 << 20) + 1)):
        with pytest.raises(sr_b200.SrError):
            sr_b200.LongStreamPool(handle, 2, mc, 2400, rate=rate)
    rate, S, c = 44100, 3, 4410
    xs = synth_at(rate, S, 24000, 0x1610)
    f = Feed(handle, xs, c, rate)
    for k in _uniform(len(xs[0]) // 2, c):
        f.push([k] * S)
    st = f.pool.state()
    with pytest.raises(sr_b200.SrError):
        f.pool.push_ragged(np.zeros((S, c + 1), np.uint16), np.array([1, c + 1, 0], np.uint32))
    with pytest.raises(sr_b200.SrError):
        f.pool.push(np.zeros((S, c + 1), np.uint16))
    st2 = f.pool.state()
    assert all(st[k].tobytes() == st2[k].tobytes() for k in st)
    while (f.n < len(xs[0])).any():                     # nothing of the refused pushes went in
        f.push(np.minimum(c, len(xs[0]) - f.n))
    f.check()
    f.close()


@pytest.mark.gpu
def test_input_count_stops_at_2_32_minus_1(handle):
    """a stream taken to 2^32 - 1 input samples at 48 kHz; n_recv is n8 of that, and the push past it fails and changes
    nothing"""
    rate, big = 48000, 1 << 20
    lim = (1 << 32) - 1
    pool = sr_b200.LongStreamPool(handle, 1, big, 0, rate=rate)
    mem, ptr = sr_b200.host_alloc_dev(0, big * 2)
    mem.view(np.uint16)[:] = 2048
    try:
        n = 0
        while n < lim:
            k = min(big, lim - n)
            assert pool.push(ptr, chunk_len=k, stride=big) == []
            n += k
        st = pool.state()
        assert int(st["n_recv"][0]) == n8(lim, rate)
        with pytest.raises(sr_b200.SrError):
            pool.push(np.full((1, 1), 2048, np.uint16))
        st2 = pool.state()
        assert all(st[k].tobytes() == st2[k].tobytes() for k in st)
        assert pool.push(np.zeros((1, 1), np.uint16)[:, :0]) == []
    finally:
        pool.close()
        sr_b200.host_free(ptr)


@pytest.mark.gpu
def test_event_buffer_footprint(handle, bank):
    """records past n_events stay as the caller left them; what did not fit comes later, per stream in order"""
    handle.set_bank(bank[0], bank[1], 4096)
    rate, S = 16000, 6
    c = rate // 100 * 8
    xs = np.array(synth_at(rate, S, 40000, 0x1620))
    ref = sr_b200.LongStreamPool(handle, S, c, 2400, rate=rate)
    pool = sr_b200.LongStreamPool(handle, S, c, 2400, rate=rate)
    buf = (sr_b200.StreamEvent * 64)()
    rec = C.sizeof(sr_b200.StreamEvent)
    all_ref, all_got = [], []
    try:
        for i, k in enumerate(_uniform(xs.shape[1], c)):
            chunk = np.full((S, c), POISON, np.uint16)
            chunk[:, :k] = xs[:, i * c:i * c + k]
            all_ref += ref.push_ragged(chunk, np.full(S, k, np.uint32))
            C.memset(buf, 0x5A, C.sizeof(buf))
            m = 1 if i % 3 else 0
            ne = pool.push_ragged(chunk, np.full(S, k, np.uint32), max_events=m, events=buf)
            assert ne <= m and bytes(buf)[ne * rec:] == b"\x5A" * (C.sizeof(buf) - ne * rec)
            all_got += pool._events(ne, buf)
        all_got += pool.fetch()
        assert len(all_got) == len(all_ref) > 10
        for s in range(S):
            assert [e for e in all_got if e["stream"] == s] == [e for e in all_ref if e["stream"] == s], s
    finally:
        ref.close()
        pool.close()


@pytest.mark.gpu
def test_two_handles_on_two_threads_equal_serial(bank):
    jobs = [(44100, synth_at(44100, 6, 20000, 0x1630)), (48000, synth_at(48000, 6, 20000, 0x1631))]

    def run(h, rate, xs):
        h.set_bank(bank[0], bank[1], 4096)
        c = rate // 100
        p = sr_b200.LongStreamPool(h, len(xs), c, 2400, rate=rate)
        evs = []
        x = np.array(xs)
        for i in range(0, x.shape[1], c):
            evs += p.push(np.ascontiguousarray(x[:, i:i + c]))
        st = p.state()
        p.close()
        return sorted((e["stream"], e["segment"]) + tuple(e[k] for k in REC) for e in evs), st["n_recv"].tolist()

    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        serial = [run(h, *j) for h, j in zip(handles, jobs)]
        assert all(len(s[0]) > 2 for s in serial)
        for rep in range(2):
            out = [None] * len(jobs)

            def work(i):
                out[i] = run(handles[i], *jobs[i])
            th = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert out == serial, rep
    finally:
        for h in handles:
            h.close()
