"""Fixed captures at any rate of SR_RESAMPLE_RATES (sr_streams_create_at_rate and sr_stream_group_create_at_rate,
include/sr_synth.h; K4 at a rate in csrc/sr_stream.cu): every push resamples each stream's chunk to 8 kHz on the GPU,
carrying the filter's history across pushes, before the capture pool's VAD and recognition.

The definition is an equivalence: after any sequence of pushes and resets, the pool at a rate is indistinguishable from
the 8 kHz pool sr_streams_create(h, S, max_samples, n_len) handed, at each push, every stream's 8 kHz outputs
[n8(before), n8(after)) as a ragged push, with n8(n) = max(0, ceil((n L - c) / M)). So every GPU test here runs the pool
beside that 8 kHz pool, fed the outputs of sr_resample_adc12_dev (K15) sliced by n8, and compares the events of every
push, sr_streams_pending and sr_streams_segments. The 8 kHz pool and K15 are pinned to their oracles by their own tests;
here K15's outputs are also checked against the numpy restatement tests/resample_ref.py where that is cheap.

CPU: the declarations and the binding; the chunk bound max_in = floor(max_samples M / L) on the restated n8.
GPU: lock-step chunks of 1, M - 1, M, M + 1, 10 ms, 80 ms and max_in at every rate, through the capture's end and past
it; ragged pushes with zero lengths; n_len 0, 2400 and 1000; resets; matchers, decision rules, the lifter and banks
switched between pushes; rate 8000 against the plain pool, launches included; refusals (rate, chunk bound, the 2^32 - 1
input count); event buffers with a canary; two handles on two threads; a group of two handles against one pool; the
digit recordings at 16, 44.1 and 48 kHz."""
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
POISON = 0xFFFF                    # past lens[s] in every chunk: a sample read from there would change the outputs
REC = ("stream", "segment", "start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


# ---- the definition, restated ---------------------------------------------------------------------------------------------
def geom(rate):
    L, M = rr.ratio(rate)
    N = len(rr.taps(rate))
    return L, M, (N - 1) // 2


def n8(n, rate):
    L, M, c = geom(rate)
    return max(0, -(-(n * L - c) // M))


def max_in(max_samples, rate):
    L, M, _ = geom(rate)
    return max_samples * M // L


def at_rate(x, rate):
    """8 kHz codes -> codes at `rate` (scipy's polyphase filter), rounded and clipped to 12 bits"""
    L, M = rr.ratio(rate)
    y = resample_poly(np.asarray(x, np.float64) - 2048, M, L)
    return np.clip(np.rint(y + 2048), 0, 4095).astype(np.uint16)


def captures(rate, S, seconds, seed):
    """S synthetic captures (300 ms of noise, then three words per 2 s) at `rate`"""
    U = int(8000 * seconds)
    return [at_rate(x, rate) for x in sr_b200.synth_pcm_host(S, U, seed, 3)]


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_header_and_binding():
    text = open(os.path.join(ROOT, "include", "sr_synth.h")).read()
    for name, commas in (("sr_streams_create_at_rate", 5), ("sr_stream_group_create_at_rate", 6)):
        decl = re.search(r"int %s\(([^;]*)\);" % name, text)
        assert decl and decl.group(1).count(",") == commas, name
        assert name not in open(os.path.join(ROOT, "include", "speech_recog.h")).read()
        assert hasattr(sr_b200.lib(), name)
    assert "max_in = floor(max_samples*M/L)" in text
    assert inspect.signature(sr_b200.StreamPool.__init__).parameters["rate"].default is None


@pytest.mark.parametrize("rate", rr.RATES)
def test_chunk_bound(rate):
    """a push of at most max_in input samples completes at most max_samples 8 kHz samples, from any input count, and
    max_in is the longest such push wherever floor and ceil differ"""
    L, M, c = geom(rate)
    a = np.arange(0, 4 * M + c + 1, dtype=np.int64)                      # every phase, past the start
    f = lambda v: np.maximum(0, -(-(v * L - c) // M))                      # noqa: E731
    assert all(n8(int(v), rate) == int(w) for v, w in zip(a[::37], f(a[::37])))
    for ms in (1, 2, 3, 79, 80, 641, 12000, 65535):
        b = max_in(ms, rate)
        small = np.arange(0, b + 1) if b < 2000 else np.array([0, 1, b - 1, b])
        for k in small:                                                    # the count grows with the chunk: b decides
            assert (f(a + k) - f(a) <= ms).all(), (rate, ms, k)
        assert (f(a + b) - f(a)).max() <= ms
        assert (f(a + b + 1) - f(a)).max() == ms + 1
    # the count of a push never falls when the chunk grows, so checking the longest chunk is checking them all
    for k in range(0, 3 * M, 7):
        assert (f(a + k + 1) - f(a) >= f(a + k) - f(a)).all()


# ---- the equivalence: a pool at a rate beside the 8 kHz pool fed K15's outputs -----------------------------------------
def k15(xs, rate):
    """sr_resample_adc12_dev on every whole recording; its first n8(n) outputs are those of the first n inputs"""
    import torch
    S, U = len(xs), max(len(x) for x in xs)
    pcm = np.full((S, U), 2048, np.uint16)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    U_out = rr.out_len(U, rate)
    x = torch.from_numpy(pcm.view(np.int16)).to("cuda:0")
    ln = torch.from_numpy(np.asarray([len(v) for v in xs], np.uint32).view(np.int32)).to("cuda:0")
    out = torch.zeros((S, U_out), dtype=torch.int16, device="cuda:0")
    st = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U, S, ln.data_ptr(), rate, out.data_ptr(), U_out, None, st.cuda_stream)
    st.synchronize()
    y = out.cpu().numpy().view(np.uint16)
    return [y[s, :n8(len(xs[s]), rate)].copy() for s in range(S)]


def by_stream(evs):
    return sorted(tuple(int(e[k]) for k in REC) for e in evs)


class Pair:
    """a pool (or group) at `rate` and the 8 kHz pool fed K15's outputs, pushed together and compared"""

    def __init__(self, h, xs, max_samples, rate, n_len=2400, handles=None, pool_rate="same"):
        self.h, self.rate = h, rate
        self.xs = [np.asarray(x, np.uint16) for x in xs]
        self.S = len(xs)
        self.max_in = max_in(max_samples, rate)
        self.pool = sr_b200.StreamPool(handles or h, self.S, max_samples, n_len,
                                       rate=rate if pool_rate == "same" else pool_rate)
        self.ref = sr_b200.StreamPool(h, self.S, max_samples, n_len)
        self.eight = k15(self.xs, rate) if rate != 8000 else [x.copy() for x in self.xs]
        self.n = np.zeros(self.S, np.int64)
        self.events = 0
        self.per_stream = np.zeros(self.S, int)

    def chunk(self, lens, width=None):
        lens = np.asarray(lens, np.int64)
        chunk = np.full((self.S, max(1, int(lens.max()) if width is None else width)), POISON, np.uint16)
        for s in range(self.S):
            assert self.n[s] + lens[s] <= len(self.xs[s])
            chunk[s, :lens[s]] = self.xs[s][self.n[s]:self.n[s] + lens[s]]
        return chunk

    def eight_chunk(self, lens):
        k0 = [n8(int(n), self.rate) for n in self.n]
        k1 = [n8(int(n + d), self.rate) for n, d in zip(self.n, lens)]
        w = np.array([b - a for a, b in zip(k0, k1)], np.uint32)
        ch = np.full((self.S, max(1, int(w.max()))), POISON, np.uint16)
        for s in range(self.S):
            ch[s, :w[s]] = self.eight[s][k0[s]:k1[s]]
        return ch, w

    def push(self, lens, lock_step=False):
        lens = np.asarray(lens, np.int64)
        ch8, w = self.eight_chunk(lens)
        if lock_step:
            assert (lens == lens[0]).all()
            got = self.pool.push(self.chunk(lens, int(lens[0]) + 3)[:, :int(lens[0])])
        else:
            got = self.pool.push_ragged(self.chunk(lens), lens.astype(np.uint32))
        want = self.ref.push_ragged(ch8, w)
        assert by_stream(got) == by_stream(want), (self.n.tolist(), lens.tolist())
        if not self.pool.group:
            assert self.pool.pending() == self.ref.pending()
        self.n += lens
        self.events += len(got)
        for e in got:
            self.per_stream[e["stream"]] += 1
        return got

    def check(self):
        sa, aa = self.pool.segments()
        sb, ab = self.ref.segments()
        assert np.array_equal(sa, sb) and aa.tobytes() == ab.tobytes()

    def reset(self):
        self.pool.reset()
        self.ref.reset()
        self.xs = [x[n:].copy() for x, n in zip(self.xs, self.n)]
        self.eight = k15(self.xs, self.rate) if self.rate != 8000 else [x.copy() for x in self.xs]
        self.n[:] = 0

    def left(self):
        return np.array([len(x) for x in self.xs]) - self.n

    def close(self):
        self.pool.close()
        self.ref.close()


def _pattern(total, pattern):
    out, n, i = [], 0, 0
    while n < total:
        out.append(min(pattern[i % len(pattern)], total - n))
        n += out[-1]
        i += 1
    return out


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bank():
    return ox.synth_bank()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", rr.RATES)
def test_lock_step_chunks(handle, bank, rate):
    """lock-step pushes cycling 1, M - 1, M, M + 1, 10 ms and 80 ms for 2 s, through a 1.5 s capture's end and past it;
    then, after a reset, pushes of max_in (1.5 s) for 2 s more"""
    handle.set_bank(bank[0], bank[1], 4096)
    L, M, _ = geom(rate)
    xs = captures(rate, 3, 4.0, 0x4A00 + rate)
    p = Pair(handle, xs, 12000, rate)
    for k in _pattern(2 * rate, [1, max(M - 1, 1), M, M + 1, rate // 100, rate // 100 * 8]):
        p.push([k] * p.S, lock_step=True)
    p.check()
    assert p.events >= 3
    p.reset()
    big = p.max_in
    while p.left().min() > 0:
        p.push([min(big, int(p.left().min()))] * p.S, lock_step=True)
    p.check()
    if rate in (16000, 48000):                                             # K15 against the numpy restatement
        assert np.array_equal(p.eight[0][:4000], rr.resample(p.xs[0][:M * 4000 + 200], rate, np.arange(4000)))
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [11025, 16000, 44100, 48000])
def test_ragged_pushes(handle, bank, rate):
    """random lengths up to max_in with zero-length streams mixed in and a late starter; captures that fill mid-push"""
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(rate)
    S, ms = 6, 8000
    p = Pair(handle, captures(rate, S, 2.0, 0x4B00), ms, rate)
    top = rate // 10
    i = 0
    while (p.left() > 0).any():
        lens = rng.integers(0, top + 1, S)
        lens[rng.random(S) < 0.25] = 0
        if i < 12:
            lens[2] = 0
        if i % 9 == 4:
            lens[rng.integers(S)] = p.max_in
        p.push(np.minimum(lens, p.left()))
        if i % 5 == 0:
            p.check()
        i += 1
    p.check()
    assert p.events >= S
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_len", [0, 2400, 1000])
def test_calibration_windows(handle, bank, n_len):
    handle.set_bank(bank[0], bank[1], 4096)
    rate = 44100
    p = Pair(handle, captures(rate, 4, 2.0, 0x4C00 + n_len), 16000, rate, n_len=n_len)
    c = rate // 100
    while (p.left() > 0).any():
        p.push(np.minimum(c, p.left()))
    p.check()
    p.close()


@pytest.mark.gpu
def test_resets_between_pushes(handle, bank):
    """a reset mid-capture restarts the input counts and the filter's history: the pool then equals a fresh 8 kHz pool
    fed what follows"""
    handle.set_bank(bank[0], bank[1], 4096)
    rate = 48000
    p = Pair(handle, captures(rate, 4, 3.0, 0x4D00), 16000, rate)
    c = rate // 100 * 3 + 17
    for cut in (int(0.7 * rate), int(1.1 * rate)):
        while p.n.min() < cut:
            p.push(np.minimum(c, p.left()))
        p.check()
        p.reset()
    while (p.left() > 0).any():
        p.push(np.minimum(c, p.left()))
    p.check()
    assert p.events >= 4
    p.close()


@pytest.mark.gpu
def test_matchers_and_banks_switched_between_pushes(handle, bank):
    bank2 = ox.synth_bank(9, 0x7E3B0000)
    rate = 22050
    configs = [(0, 0, bank), (sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE | sr_b200.dtw_reject(30), 118, bank2),
               (sr_b200.dtw_knn(2) | sr_b200.DTW_LIFTER, 0, bank), (sr_b200.DTW_SYM_P1 | sr_b200.DTW_LIFTER, 10, bank2),
               (sr_b200.dtw_reject(80), 0, bank2)]
    p = Pair(handle, captures(rate, 6, 2.0, 0x4E00), 16000, rate)
    rng = np.random.default_rng(5)
    c = rate // 100 * 4
    try:
        while (p.left() > 0).any():
            flags, r, b = configs[int(rng.integers(len(configs)))]
            handle.set_match(flags, r)
            handle.set_bank(b[0], b[1], 4096)
            p.push(np.minimum(c, p.left()))
        p.check()
        assert p.events >= 6
    finally:
        handle.set_match(0, 0)
    p.close()


@pytest.mark.gpu
def test_8000_is_the_plain_pool(handle, bank):
    """rate 8000: the pool sr_streams_create makes -- events, segments and launches, push for push"""
    handle.set_bank(bank[0], bank[1], 4096)
    rng = np.random.default_rng(8)
    p = Pair(handle, captures(8000, 5, 2.0, 0x4F00), 12000, 8000)
    assert p.max_in == 12000
    while (p.left() > 0).any():
        lens = np.minimum(rng.integers(0, 1200, p.S), p.left())
        l0 = handle.launch_count()
        a = p.pool.push_ragged(p.chunk(lens), lens.astype(np.uint32))
        l1 = handle.launch_count()
        b = p.ref.push_ragged(p.chunk(lens), lens.astype(np.uint32))
        assert l1 - l0 == handle.launch_count() - l1
        assert by_stream(a) == by_stream(b)
        p.n += lens
    p.check()
    l0 = handle.launch_count()
    p.pool.reset()
    l1 = handle.launch_count()
    p.ref.reset()
    assert l1 - l0 == handle.launch_count() - l1
    p.close()


@pytest.mark.gpu
def test_one_launch_more_than_at_8000(handle, bank):
    rate, S = 44100, 8
    c = rate // 100
    xs = np.array(captures(rate, S, 0.5, 0x5000))
    pool = sr_b200.StreamPool(handle, S, 16000, 2400, rate=rate)
    plain = sr_b200.StreamPool(handle, S, 16000, 2400)
    try:
        for with_bank in (True, False):
            handle.set_bank(*((bank[0], bank[1]) if with_bank else (np.zeros((0, 4096), np.uint8), 0)), 4096)
            for i in range(0, xs.shape[1] - c, 7 * c):
                before = handle.launch_count()
                pool.push(np.ascontiguousarray(xs[:, i:i + c]))
                mid = handle.launch_count()
                plain.push(np.ascontiguousarray(xs[:, i:i + 80]))
                assert mid - before == handle.launch_count() - mid + 1
    finally:
        pool.close()
        plain.close()


@pytest.mark.gpu
def test_refusals_write_nothing(handle, bank):
    """a bad rate is refused before anything exists; a chunk over max_in is refused before any stream changes, with no
    launch and no event record written, and the pool carries on as if it had not been tried"""
    handle.set_bank(bank[0], bank[1], 4096)
    for rate in (0, 7999, 12000, 44000, 96000):
        l0 = handle.launch_count()
        with pytest.raises(sr_b200.SrError):
            sr_b200.StreamPool(handle, 2, 8000, 2400, rate=rate)
        with pytest.raises(sr_b200.SrError):
            sr_b200.StreamPool([handle, handle], 2, 8000, 2400, rate=rate)
        assert handle.launch_count() == l0
    with pytest.raises(sr_b200.SrError):
        sr_b200.StreamPool(handle, 2, 65536, 2400, rate=48000)
    rate, S = 44100, 3
    p = Pair(handle, captures(rate, S, 1.5, 0x5100), 8000, rate)
    assert p.max_in == 8000 * 441 // 80
    c = rate // 100
    for _ in range(30):
        p.push([c] * S)
    seg0 = p.pool.segments()
    for bad in (np.array([1, p.max_in + 1, 0]), np.array([p.max_in + 1] * S)):
        C.memset(p.pool._ev, 0x5A, C.sizeof(p.pool._ev))
        l0 = handle.launch_count()
        with pytest.raises(sr_b200.SrError):
            if (bad == bad[0]).all():
                p.pool.push(np.zeros((S, int(bad[0])), np.uint16))
            else:
                p.pool.push_ragged(np.zeros((S, int(bad.max())), np.uint16), bad.astype(np.uint32))
        assert handle.launch_count() == l0
        assert bytes(p.pool._ev) == b"\x5A" * C.sizeof(p.pool._ev)
    seg1 = p.pool.segments()
    assert np.array_equal(seg0[0], seg1[0]) and seg0[1].tobytes() == seg1[1].tobytes()
    while (p.left() > 0).any():
        p.push(np.minimum(c, p.left()))
    p.check()
    p.close()


@pytest.mark.gpu
def test_input_count_stops_at_2_32_minus_1(handle):
    """a stream taken to 2^32 - 1 input samples at 48 kHz in pushes of max_in from pinned memory; the push past it fails
    and changes nothing, a push of nothing still works, and a reset starts the count again"""
    rate, ms = 48000, 65535
    big, lim = max_in(ms, rate), (1 << 32) - 1
    pool = sr_b200.StreamPool(handle, 1, ms, 2400, rate=rate)
    mem, ptr = sr_b200.host_alloc_dev(0, big * 2)
    mem.view(np.uint16)[:] = 2048
    try:
        n = 0
        while n < lim:
            k = min(big, lim - n)
            assert pool.push(ptr, chunk_len=k, stride=big) == []
            n += k
        seg = pool.segments()
        l0 = handle.launch_count()
        with pytest.raises(sr_b200.SrError):
            pool.push(np.full((1, 1), 2048, np.uint16))
        assert handle.launch_count() == l0
        seg2 = pool.segments()
        assert np.array_equal(seg[0], seg2[0]) and seg[1].tobytes() == seg2[1].tobytes()
        assert pool.push(np.zeros((1, 1), np.uint16)[:, :0]) == []
        pool.reset()
        assert pool.push(ptr, chunk_len=big, stride=big) == []
    finally:
        pool.close()
        sr_b200.host_free(ptr)


@pytest.mark.gpu
def test_event_buffers_with_a_canary(handle, bank):
    """only n_events records are written; what did not fit comes out by the next push or by fetch, per stream in order,
    and sr_streams_pending agrees with the 8 kHz pool"""
    handle.set_bank(bank[0], bank[1], 4096)
    rate, S = 16000, 6
    p = Pair(handle, captures(rate, S, 2.0, 0x5200), 16000, rate)
    L = sr_b200.lib()
    buf = (sr_b200.StreamEvent * 64)()
    rec = C.sizeof(sr_b200.StreamEvent)
    got, want = [], []
    c = rate // 100 * 8
    i = peak = 0
    while (p.left() > 0).any():
        lens = np.minimum(c, p.left())
        ch8, w = p.eight_chunk(lens)
        m = 1 if i % 3 else 0
        ne, ne8 = C.c_uint32(0), C.c_uint32(0)
        C.memset(buf, 0x5A, C.sizeof(buf))
        ch, ln = p.chunk(lens), np.ascontiguousarray(lens, np.uint32)
        assert L.sr_streams_push_ragged(p.pool._p, ch.ctypes.data_as(C.c_void_p), ch.shape[1], ln.ctypes.data_as(C.c_void_p),
                                        buf, m, C.byref(ne)) == 0
        assert ne.value <= m and bytes(buf)[ne.value * rec:] == b"\x5A" * (C.sizeof(buf) - ne.value * rec)
        got += [{k: getattr(buf[j], k) for k in REC} for j in range(ne.value)]
        buf8 = (sr_b200.StreamEvent * 64)()
        assert L.sr_streams_push_ragged(p.ref._p, ch8.ctypes.data_as(C.c_void_p), ch8.shape[1], w.ctypes.data_as(C.c_void_p),
                                        buf8, m, C.byref(ne8)) == 0
        assert ne.value == ne8.value and p.pool.pending() == p.ref.pending()
        peak = max(peak, p.pool.pending())
        want += [{k: getattr(buf8[j], k) for k in REC} for j in range(ne8.value)]
        p.n += lens
        i += 1
    assert peak > 0
    got += p.pool.fetch()
    want += p.ref.fetch()
    assert p.pool.pending() == 0
    assert len(got) == len(want) >= S
    for s in range(S):
        assert [by_stream([e]) for e in got if e["stream"] == s] == [by_stream([e]) for e in want if e["stream"] == s]
    p.close()


@pytest.mark.gpu
def test_two_handles_on_two_threads_equal_serial(bank):
    jobs = [(44100, captures(44100, 5, 2.0, 0x5300)), (48000, captures(48000, 5, 2.0, 0x5301))]

    def run(h, rate, xs):
        h.set_bank(bank[0], bank[1], 4096)
        c = rate // 100
        pool = sr_b200.StreamPool(h, len(xs), 16000, 2400, rate=rate)
        x = np.array(xs)
        evs = []
        for i in range(0, x.shape[1] - c + 1, c):
            evs += pool.push(np.ascontiguousarray(x[:, i:i + c]))
        seg = pool.segments()[0]
        pool.close()
        return by_stream(evs), seg.tolist()

    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        serial = [run(h, *j) for h, j in zip(handles, jobs)]
        assert all(len(s[0]) >= 5 for s in serial)
        out = [None] * len(jobs)

        def work(i):
            out[i] = run(handles[i], *jobs[i])
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert out == serial
    finally:
        for h in handles:
            h.close()


@pytest.mark.gpu
def test_group_of_two_handles_equals_one_pool(bank):
    """a group at a rate over two handles of device 0 against the 8 kHz pool with all the streams; lens and chunk by
    global stream"""
    handles = [sr_b200.Handle(0) for _ in range(2)]
    try:
        for h in handles:
            h.set_bank(bank[0], bank[1], 4096)
        rate, S = 44100, 7
        p = Pair(handles[0], captures(rate, S, 2.0, 0x5400), 12000, rate, handles=handles)
        rng = np.random.default_rng(11)
        while (p.left() > 0).any():
            lens = rng.integers(0, rate // 20, S)
            lens[rng.random(S) < 0.2] = 0
            p.push(np.minimum(lens, p.left()))
        p.check()
        assert p.events >= S
        p.close()
    finally:
        for h in handles:
            h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_digit_recordings(handle, rate):
    """the four digit recordings taken to `rate` and fed in 10 ms chunks: every push equals the 8 kHz pool fed K15's
    outputs, and K15's outputs equal the numpy restatement"""
    lo, port = ox.long_oracle(), ob.port()
    from cases import digit_bank
    bk, T, _ = digit_bank(port, lo, ox.golden_wav(DIGITS[1]))
    handle.set_bank(bk, T, 4096)
    xs = [at_rate(ox.golden_wav(n), rate) for n in DIGITS]
    p = Pair(handle, xs, 65535, rate)
    c = rate // 100
    while (p.left() > 0).any():
        p.push(np.minimum(c, p.left()))
    p.check()
    s = 2
    k = min(len(p.eight[s]), 16000)
    assert np.array_equal(p.eight[s][:k], rr.resample(p.xs[s], rate, np.arange(k)))
    print("K4 at %d Hz, digit recordings in 10 ms chunks: %d events, per capture %s" % (rate, p.events, p.per_stream.tolist()))
    assert p.events > 0
    p.close()
