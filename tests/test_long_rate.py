"""The host-buffer long-form calls at any rate of SR_RESAMPLE_RATES (sr_recognise_long_batch_at_rate and
sr_recognise_long_grammar_batch_at_rate, include/sr_synth.h): recordings in host memory at 16, 44.1 or 48 kHz, staged in
groups of at most 256 MB of input and resampled to 8 kHz on the GPU group by group.

The definition is an equivalence: the call writes exactly what the 8 kHz call writes on y_b, the ceil(len_b L / M)
outputs of sr_resample_adc12_dev on each recording's first len_b samples, at stride U8 = ceil(U_in L / M) with
lens8[b] = ceil(len_b L / M). So every GPU test here compares the call with sr_resample_adc12_dev, a copy back and the
8 kHz host call (both pinned to their oracles elsewhere), and a few with the CPU composition tests/resample_ref.py + the
long-form oracles, which also holds K15's lengths to the ceiling.

CPU: the header and the binding, U8 / lens8 against tests/resample_ref.py at edge lengths, and the grouping rule restated.
GPU: every rate with ragged lengths (0, 1, around one 8 kHz frame, the calibration edge) and lens = NULL; max_segs and
max_words below the counts; atap NULL and in / out; every output pointer NULL in turn with canaries around every buffer;
the four matchers, the decision rules, the lifter and SR_GEOM_B; the loop and a digit-string grammar; the digit
recordings; rate 8000 against the 8 kHz call (bytes, launches, tags); launches and tags at other rates; refusals; three
staging groups and one recording over 256 MB; two handles on two threads."""
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
GROUP_BYTES = 256 << 20            # kLongGroupBytes, csrc/sr_api.cu: input PCM per staged group
LONG_U_MAX = 1 << 27               # SR_LONG_U_MAX
RESAMPLE_U_MAX = 1 << 30           # SR_RESAMPLE_U_MAX
TAG_RESAMPLE = 15
RATES = [r for r in rr.RATES if r != 8000]
LOOP = sr_b200.loop_grammar()
DIGIT_STRING = sr_b200.chain_grammar(3, 0x3FF)
CANARY = 0xA5
PAD = 64                           # canary bytes before and after every output buffer


# ---- the definition, restated ---------------------------------------------------------------------------------------------
def u8(n, rate):
    """ceil(n L / M): U8 of a row of n input samples, and lens8 of a recording of n samples"""
    L, M = rr.ratio(rate)
    return -(-n * L // M)


def group_size(U_in, B):
    """recordings per staged group: whole recordings, at most GROUP_BYTES of input unless the group holds one"""
    return max(1, min(GROUP_BYTES // (2 * U_in), B))


def n_groups(U_in, B):
    return -(-B // group_size(U_in, B))


def at_rate(x, rate):
    """8 kHz codes -> codes at `rate` (scipy's polyphase filter), rounded and clipped to 12 bits"""
    L, M = rr.ratio(rate)
    y = resample_poly(np.asarray(x, np.float64) - 2048, M, L)
    return np.clip(np.rint(y + 2048), 0, 4095).astype(np.uint16)


def cal_edge(rate, n_len=2400):
    """the longest input whose ceil(len L / M) is n_len while its floor is n_len - 1: calibration runs on the ceiling"""
    L, M = rr.ratio(rate)
    return -(-n_len * M // L) - 1


def batch_at(rate, lens, seed, U_in=None):
    """recordings at `rate` of the given input lengths (many words each), rows of U_in samples poisoned past each length"""
    lens = np.asarray(lens, np.int64)
    U_in = int(lens.max()) if U_in is None else U_in
    L, M = rr.ratio(rate)
    xs = ox.synth_long(len(lens), u8(U_in, rate) + 64, seed)
    pcm = np.zeros((len(lens), U_in), np.uint16)
    for b in range(len(lens)):
        pcm[b] = at_rate(xs[b], rate)[:U_in]
        pcm[b, lens[b]:] = np.where(np.arange(U_in - lens[b]) % 2, 4095, 0)
    return pcm


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_header_and_binding():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sr_synth.h")).read(), flags=re.S)
    d1 = re.search(r"int sr_recognise_long_batch_at_rate\(([^;]*)\);", text)
    d2 = re.search(r"int sr_recognise_long_grammar_batch_at_rate\(([^;]*)\);", text)
    assert d1 and d1.group(1).count(",") == 8 and d2 and d2.group(1).count(",") == 11
    assert '#include "sr_long_grammar.h"' in text and "sr_long_gram_out *out" in text
    for h in ("sr_long.h", "sr_long_grammar.h"):
        assert "_at_rate" not in open(os.path.join(ROOT, "include", h)).read()
    assert "15 the resampling" in open(os.path.join(ROOT, "include", "speech_recog.h")).read()
    L = sr_b200.lib()
    assert hasattr(L, "sr_recognise_long_batch_at_rate") and hasattr(L, "sr_recognise_long_grammar_batch_at_rate")
    for m in (sr_b200.Handle.recognise_long_batch, sr_b200.Handle.recognise_long_grammar):
        assert inspect.signature(m).parameters["rate"].default is None


@pytest.mark.parametrize("rate", rr.RATES)
def test_u8_and_lens8_match_resample_ref(rate):
    L, M = rr.ratio(rate)
    rng = np.random.default_rng(rate)
    for n in (0, 1, M - 1, M, M + 1, 2 * M - 1, 159, 160, 161, cal_edge(rate) if rate != 8000 else 2399, 12345):
        assert u8(n, rate) == rr.out_len(n, rate), n
        x = rng.integers(0, 4096, n).astype(np.uint16)
        assert len(rr.resample(x, rate)) == u8(n, rate), n
    # the SR_LONG_U_MAX boundary: the longest row the calls take, and one sample more
    top = LONG_U_MAX * M // L
    assert u8(top, rate) <= LONG_U_MAX < u8(top + 1, rate)
    assert rr.out_len(top, rate) == u8(top, rate) and rr.out_len(top + 1, rate) == u8(top + 1, rate)
    assert top <= RESAMPLE_U_MAX
    if rate != 8000:
        assert u8(cal_edge(rate), rate) == 2400 and cal_edge(rate) * L // M == 2399


def test_grouping_rule():
    """the counts the GPU tests below check through the tag-15 records"""
    assert n_groups(48000 * 9, 6) == 1 and n_groups(44100 * 9, 7) == 1
    half_hour = 48000 * 1800
    assert half_hour * 2 == 172800000 and group_size(half_hour, 3) == 1 and n_groups(half_hour, 3) == 3
    assert n_groups(140_000_000, 1) == 1 and 140_000_000 * 2 > GROUP_BYTES
    # by 8 kHz bytes all three half-hour recordings would share one group
    assert max(1, min(GROUP_BYTES // (2 * u8(half_hour, 48000)), 3)) == 3
    assert group_size(1, 1 << 30) == 1 << 27 and group_size(GROUP_BYTES // 2 + 1, 5) == 1


# ---- the reference: sr_resample_adc12_dev, a copy back, the 8 kHz host call -------------------------------------------------
def gpu_eight(pcm, lens, rate):
    """(y [B, U8], lens8 [B]) from sr_resample_adc12_dev on the rows of pcm (lens None: U_in each)"""
    import torch
    B, U_in = pcm.shape
    U8 = u8(U_in, rate)
    x = torch.from_numpy(pcm.view(np.int16)).to("cuda:0")
    ln = None if lens is None else torch.from_numpy(np.asarray(lens, np.uint32).view(np.int32)).to("cuda:0")
    out = torch.zeros((B, max(U8, 1)), dtype=torch.int16, device="cuda:0")
    ol = torch.zeros(B, dtype=torch.int32, device="cuda:0")
    s0 = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U_in, B, None if ln is None else ln.data_ptr(), rate, out.data_ptr(), U8,
                               ol.data_ptr(), s0.cuda_stream)
    s0.synchronize()
    y = np.ascontiguousarray(out.cpu().numpy().view(np.uint16)[:, :U8])
    return y, ol.cpu().numpy().view(np.uint32).copy()


def cpu_eight(pcm, lens, rate):
    B, U_in = pcm.shape
    lens = np.full(B, U_in, np.uint32) if lens is None else np.asarray(lens, np.uint32)
    y = rr.resample_batch(pcm, rate, lens, u8(U_in, rate))
    return y, np.array([u8(int(n), rate) for n in lens], np.uint32)


def cmp_long(got, want, max_segs):
    assert got["atap"].tobytes() == want["atap"].tobytes()
    assert got["n_segs"].tolist() == want["n_segs"].tolist()
    for b in range(len(want["n_segs"])):
        m = min(int(want["n_segs"][b]), max_segs)
        assert got["segs"][b, :m].tobytes() == want["segs"][b, :m].tobytes(), b


def cmp_gram(got, want, max_segs, max_words):
    for b in range(len(want["n_segs"])):
        assert got["atap"][b].tobytes() == want["atap"][b].tobytes(), b
        assert int(got["n_segs"][b]) == int(want["n_segs"][b]), b
        m = min(int(want["n_segs"][b]), max_segs)
        for k in ("seg_off", "frm_num", "seg_status"):
            assert got[k][b, :m].tobytes() == want[k][b, :m].tobytes(), (b, k)
        assert int(got["n_words"][b]) == int(want["n_words"][b]) and int(got["total"][b]) == int(want["total"][b]), b
        m = min(int(want["n_words"][b]), max_words)
        assert got["words"][b, :m].tobytes() == want["words"][b, :m].tobytes(), b


def long_pair(h, pcm, lens, rate, max_segs, n_len=2400, atap=None):
    """(the call at `rate`, the composition) with the same prefilled outputs: every byte must agree"""
    B = pcm.shape[0]
    at = np.zeros(B, sr_b200.ATAP_DTYPE) if atap is None else atap
    fill = np.frombuffer(bytes([CANARY]) * (B * max_segs * 28), sr_b200.LONG_SEG_DTYPE).reshape(B, max_segs)
    got = h.recognise_long_batch(pcm, max_segs, n_len, lens, at.copy(), fill.copy(), rate=rate)
    y, l8 = gpu_eight(pcm, lens, rate)
    want = h.recognise_long_batch(y, max_segs, n_len, l8, at.copy(), fill.copy())
    for k in got:
        assert got[k].tobytes() == want[k].tobytes(), k
    return got, (y, l8)


def gram_out(B, max_segs, max_words, atap=None, want=sr_b200.LONG_GRAM_FIELDS):
    out = {"atap": np.zeros(B, ob.ATAP_DTYPE) if atap is None else atap.copy(),
           "n_segs": np.full(B, 0xA5A5A5A5, np.uint32), "seg_off": np.full((B, max_segs, 2), 0xA5A5A5A5, np.uint32),
           "frm_num": np.full((B, max_segs), 0xA5A5A5A5, np.uint32), "seg_status": np.full((B, max_segs), CANARY, np.uint8),
           "n_words": np.full(B, 0xA5A5A5A5, np.uint32),
           "words": np.frombuffer(bytes([CANARY]) * (B * max_words * 24), sr_b200.WORD_DTYPE).copy().reshape(B, max_words),
           "total": np.full(B, 0xA5A5A5A5A5A5A5A5, np.uint64)}
    return {k: v for k, v in out.items() if k in want}


def gram_pair(h, pcm, lens, rate, g, max_segs, max_words, n_len=2400, atap=None, penalty=1000, want=sr_b200.LONG_GRAM_FIELDS):
    B = pcm.shape[0]
    got = h.recognise_long_grammar(pcm, g, penalty, max_segs, max_words, n_len, lens,
                                   out=gram_out(B, max_segs, max_words, atap, want), rate=rate)
    y, l8 = gpu_eight(pcm, lens, rate)
    ref = h.recognise_long_grammar(y, g, penalty, max_segs, max_words, n_len, l8, out=gram_out(B, max_segs, max_words, atap, want))
    for k in ref:
        assert got[k].tobytes() == ref[k].tobytes(), k
    return got, (y, l8)


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bank():
    return ox.synth_bank()


def ragged(rate):
    """input lengths: 0, 1, 159 and 161 outputs (around one 8 kHz frame), the calibration edge, a long one, a full row"""
    L, M = rr.ratio(rate)
    U_in = rate * 9
    return U_in, np.array([0, 1, 159 * M // L, 161 * M // L + 1, cal_edge(rate), U_in - 3, U_in], np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
def test_every_rate_ragged_equals_composition(handle, bank, rate):
    """both calls at every rate: ragged lengths, lens = NULL, max_segs and max_words below the counts, a prefilled atap"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    U_in, lens = ragged(rate)
    pcm = batch_at(rate, lens, 0x1A00 + rate, U_in)
    atap = np.zeros(len(lens), sr_b200.ATAP_DTYPE)
    atap.view(np.uint8)[:] = 0x3C                     # stays where noise_atap does not run (lens8 < n_len)
    got, _ = long_pair(handle, pcm, lens, rate, 64, atap=atap)
    ns = got["n_segs"]
    assert ns[-1] > 3 and (ns[:2] == 0).all()
    assert got["atap"][4].tobytes() != atap[4].tobytes()     # calibrated: lens8 is the ceiling, n_len = 2400
    long_pair(handle, pcm, lens, rate, 1, atap=atap)
    long_pair(handle, pcm, lens, rate, 0)
    long_pair(handle, pcm, lens, rate, max(1, int(ns.max()) - 2), n_len=0)
    long_pair(handle, pcm[4:], None, rate, 32)
    gram, _ = gram_pair(handle, pcm, lens, rate, LOOP, 64, 256, atap=atap)
    assert int(gram["n_words"].max()) > 3
    gram_pair(handle, pcm, lens, rate, DIGIT_STRING, 2, max(1, int(gram["n_words"].max()) - 2))
    gram_pair(handle, pcm[4:], None, rate, LOOP, 0, 0)


@pytest.mark.gpu
def test_three_groups_and_one_over_256_mb():
    """three half-hour recordings at 48 kHz (173 MB each: one per group, of different lengths), then one recording of
    280 MB at 48 kHz alone in its group: the groups counted by the tag-15 records, every byte equal to the composition"""
    h = sr_b200.Handle(0)
    try:
        h.set_bank(*ox.synth_bank(), 4096)
        rate, U_in = 48000, 48000 * 1800
        lens = np.array([U_in, U_in - 12345, U_in - 777777], np.uint32)
        base = ox.synth_long(3, u8(U_in, rate), 0x1A70)
        pcm = np.repeat(base, 6, axis=1)[:, :U_in]
        for b in range(3):
            pcm[b, lens[b]:] = 4095
        assert n_groups(U_in, 3) == 3
        h.timing_enable(4096)
        h.timing_collect()
        got, _ = long_pair(h, pcm, lens, rate, 512)
        tags = [t for t, _ in h.timing_collect()]
        assert tags.count(TAG_RESAMPLE) == 3 and int(got["n_segs"].min()) > 100
        gram_pair(h, pcm, lens, rate, LOOP, 512, 2048)
        tags = [t for t, _ in h.timing_collect()]
        assert tags.count(TAG_RESAMPLE) == 3
        del pcm, base
        U_big = 140_000_000
        assert n_groups(U_big, 1) == 1 and U_big * 2 > GROUP_BYTES
        big = np.ascontiguousarray(np.repeat(ox.synth_long(1, u8(U_big, rate) + 1, 0x1A71), 6, axis=1)[:, :U_big])
        got, _ = long_pair(h, big, None, rate, 64)
        tags = [t for t, _ in h.timing_collect()]
        assert tags.count(TAG_RESAMPLE) == 1 and int(got["n_segs"][0]) > 64
        h.timing_enable(0)
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [11025, 44100, 48000])
def test_cpu_oracle_composition(handle, bank, rate):
    """resample_ref, then the long-form oracles: this also holds K15's lengths (lens8) to the ceiling"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    L, M = rr.ratio(rate)
    U_in = rate * 5
    lens = np.array([cal_edge(rate), U_in - 1, 161 * M // L + 1, U_in], np.uint32)
    pcm = batch_at(rate, lens, 0x1A10 + rate, U_in)
    y, l8 = cpu_eight(pcm, lens, rate)
    gy, gl8 = gpu_eight(pcm, lens, rate)
    assert gl8.tolist() == l8.tolist()
    for b in range(len(lens)):
        assert gy[b, :l8[b]].tobytes() == y[b, :l8[b]].tobytes(), b
    lo, port, lg = ox.long_oracle(), ob.port(), ox.long_grammar()
    got = handle.recognise_long_batch(pcm, 32, 2400, lens, rate=rate)
    want = ox.recognise_long(lo, port, y, 2400, bank[0], bank[1], 4096, 32, l8)
    cmp_long(got, want, 32)
    assert int(got["n_segs"].sum()) > 6
    gg = handle.recognise_long_grammar(pcm, DIGIT_STRING, 1000, 32, 64, 2400, lens, rate=rate)
    gw = ox.recognise_long_grammar(lo, port, lg, y, 2400, bank[0], bank[1], 4096, DIGIT_STRING, 1000, 32, 64, l8)
    cmp_gram(gg, gw, 32, 64)


@pytest.mark.gpu
def test_rate_8000_is_the_8khz_call(handle, bank):
    """the same bytes, launch counts and timing tags as the 8 kHz calls, and no resample launch"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    lens = np.array([0, 1, 2399, 2400, 60000, 72000], np.uint32)
    pcm = batch_at(8000, lens, 0x1A20)
    handle.timing_enable(4096)
    handle.timing_collect()
    runs = []
    for rate in (8000, None):
        c0 = handle.launch_count()
        a = handle.recognise_long_batch(pcm, 16, 2400, lens, rate=rate)
        g = handle.recognise_long_grammar(pcm, LOOP, 1000, 16, 64, 2400, lens, rate=rate)
        runs.append((handle.launch_count() - c0, [t for t, _ in handle.timing_collect()], a, g))
    (n0, t0, a0, g0), (n1, t1, a1, g1) = runs
    assert n0 == n1 and t0 == t1 and TAG_RESAMPLE not in t0
    for k in a0:
        assert a0[k].tobytes() == a1[k].tobytes(), k
    for k in g0:
        assert g0[k].tobytes() == g1[k].tobytes(), k
    handle.timing_enable(0)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100])
def test_launches_and_tags_at_a_rate(handle, bank, rate):
    """one group: the 8 kHz call's launches and tags with one resample launch, tag 15, first"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    U_in, lens = ragged(rate)
    pcm = batch_at(rate, lens, 0x1A30 + rate, U_in)
    y, l8 = gpu_eight(pcm, lens, rate)
    assert n_groups(U_in, len(lens)) == 1
    handle.timing_enable(4096)
    handle.timing_collect()
    for call in (lambda x, ln, r: handle.recognise_long_batch(x, 16, 2400, ln, rate=r),
                 lambda x, ln, r: handle.recognise_long_grammar(x, LOOP, 1000, 16, 64, 2400, ln, rate=r)):
        c0 = handle.launch_count()
        call(pcm, lens, rate)
        n_rate, t_rate = handle.launch_count() - c0, [t for t, _ in handle.timing_collect()]
        c0 = handle.launch_count()
        call(y, l8, None)
        n_8k, t_8k = handle.launch_count() - c0, [t for t, _ in handle.timing_collect()]
        assert n_rate == n_8k + 1 and t_rate == [TAG_RESAMPLE] + t_8k
    handle.timing_enable(0)


MATCHERS = [(0, 0), (sr_b200.DTW_BAND, 10), (sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE, 118),
            (sr_b200.DTW_SYM_P1, 10),
            (sr_b200.DTW_BAND | sr_b200.DTW_LIFTER | sr_b200.dtw_knn(3) | sr_b200.dtw_reject(100), 10)]


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_matchers_rules_and_geometry(handle, bank, geom):
    handle.set_bank(bank[0], bank[1], 4096)
    rate = 44100
    U_in, lens = ragged(rate)
    pcm = batch_at(rate, lens, 0x1A40, U_in)
    handle.set_geometry(geom)
    try:
        for flags, r in MATCHERS:
            handle.set_match(flags, r)
            got, _ = long_pair(handle, pcm, lens, rate, 32)
            assert int(got["n_segs"].sum()) > 6
        handle.set_match(0, 0)
        gram_pair(handle, pcm, lens, rate, DIGIT_STRING, 32, 64)
    finally:
        handle.set_match(0, 0)
        handle.set_geometry(0)


def _raw_long(h, fn, pcm, lens, rate, max_segs, null):
    """one raw call of fn (the 8 kHz call when rate is None) with the outputs named in null passed as NULL and PAD canary
    bytes before and after every other buffer: the buffers, canaries included"""
    B, U = pcm.shape
    sizes = {"atap": B * 12, "n_segs": B * 4, "segs": B * max_segs * 28}
    bufs = {k: np.full(n + 2 * PAD, CANARY, np.uint8) for k, n in sizes.items()}
    bufs["atap"][PAD:PAD + B * 12] = 0
    ptr = {k: None if (k in null or (k == "segs" and max_segs == 0)) else bufs[k].ctypes.data + PAD for k in sizes}
    out = sr_b200.LongOut(ptr["atap"], ptr["n_segs"], ptr["segs"])
    ln = None if lens is None else np.ascontiguousarray(lens, np.uint32)
    lp = None if ln is None else ln.ctypes.data
    if rate is None:
        rc = fn(h._h, pcm.ctypes.data, U, B, lp, 2400, max_segs, C.byref(out))
    else:
        rc = fn(h._h, pcm.ctypes.data, U, B, lp, rate, 2400, max_segs, C.byref(out))
    assert rc == 0
    for k in sizes:
        assert set(bufs[k][:PAD].tobytes()) == {CANARY} and set(bufs[k][PAD + sizes[k]:].tobytes()) == {CANARY}, k
        if ptr[k] is None:
            assert set(bufs[k][PAD:PAD + sizes[k]].tobytes()) <= {CANARY, 0}, k
    return bufs


@pytest.mark.gpu
def test_null_outputs_and_footprint(handle, bank):
    """every output pointer NULL in turn (atap NULL included), canaries around every buffer: the call at a rate writes the
    bytes the composition writes, and nothing else"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 48000
    U_in, lens = ragged(rate)
    pcm = batch_at(rate, lens, 0x1A50, U_in)
    y, l8 = gpu_eight(pcm, lens, rate)
    L = sr_b200.lib()
    for max_segs in (0, 3, 40):
        for null in ((), ("atap",), ("n_segs",), ("segs",), ("atap", "n_segs", "segs")):
            if "segs" in null and max_segs:
                continue                               # segs may be NULL only when max_segs = 0
            a = _raw_long(handle, L.sr_recognise_long_batch_at_rate, pcm, lens, rate, max_segs, null)
            b = _raw_long(handle, L.sr_recognise_long_batch, y, l8, None, max_segs, null)
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), (max_segs, null, k)
    # the grammar call: each output NULL in turn, canaries in every record past what the composition writes
    for drop in sr_b200.LONG_GRAM_FIELDS:
        want = tuple(k for k in sr_b200.LONG_GRAM_FIELDS if k != drop)
        gram_pair(handle, pcm, lens, rate, LOOP, 5, 7, want=want)
    got, _ = gram_pair(handle, pcm, lens, rate, LOOP, 5, 7)
    for b in range(len(lens)):
        m = min(int(got["n_segs"][b]), 5)
        assert set(got["seg_off"][b, m:].tobytes()) <= {CANARY} and set(got["frm_num"][b, m:].tobytes()) <= {CANARY}
        assert set(got["words"][b, min(int(got["n_words"][b]), 7):].tobytes()) <= {CANARY}


@pytest.mark.gpu
def test_refusals_write_nothing(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 44100
    U_in, lens = ragged(rate)
    pcm = batch_at(rate, lens, 0x1A60, U_in)
    B = len(lens)
    bad_lens = lens.copy()
    bad_lens[3] = U_in + 1
    top = LONG_U_MAX * 441 // 80                        # the longest row at 44.1 kHz
    big = np.zeros((1, top + 1), np.uint16)
    cases = [dict(rate=0), dict(rate=7999), dict(rate=12000), dict(rate=96000), dict(lens=bad_lens),
             dict(n_len=65536), dict(pcm=big[:, :top + 1], lens=None), dict(max_segs=(1 << 32) // B + 1, lens=None)]
    for c in cases:
        x, ln, r, n_len = c.get("pcm", pcm), c.get("lens", lens), c.get("rate", rate), c.get("n_len", 2400)
        ms = c.get("max_segs", 4)
        n = x.shape[0]
        segs = np.frombuffer(bytes([CANARY]) * (n * min(ms, 4) * 28), sr_b200.LONG_SEG_DTYPE).copy().reshape(n, min(ms, 4))
        at = np.frombuffer(bytes([CANARY]) * (n * 12), sr_b200.ATAP_DTYPE).copy()
        l0 = handle.launch_count()
        with pytest.raises(sr_b200.SrError):
            if ms > 4:                                 # too many slots: passed raw, so no buffer of that size is needed
                out = sr_b200.LongOut(at.ctypes.data, None, segs.ctypes.data)
                handle._ck(sr_b200.lib().sr_recognise_long_batch_at_rate(handle._h, x.ctypes.data, x.shape[1], n, None, r,
                                                                         n_len, ms, C.byref(out)))
            else:
                handle.recognise_long_batch(x, ms, n_len, ln, at, segs, rate=r)
        assert set(segs.tobytes()) == {CANARY} and set(at.tobytes()) == {CANARY}, c
        out = gram_out(n, 4, 4, at)
        with pytest.raises(sr_b200.SrError):
            handle.recognise_long_grammar(x, LOOP, 1000, 4, 4, n_len, ln, out=out, rate=r) if ms <= 4 else \
                handle._ck(sr_b200.lib().sr_recognise_long_grammar_batch_at_rate(
                    handle._h, x.ctypes.data, x.shape[1], n, None, r, n_len, None, 0, ms, 4,
                    C.byref(sr_b200.LongGramOut(*[None] * 8))))
        for k, v in out.items():
            assert set(np.asarray(v).tobytes()) <= {CANARY}, (c, k)
        assert handle.launch_count() == l0, c
    # grammars the 8 kHz call refuses: malformed, and more copies than SR_GRAM_COPY_MAX
    too_long, too_wide = sr_b200.chain_grammar(20, 0xFFF), sr_b200.chain_grammar(12, 0xFFF)   # 21 states; 144 copies
    for g in ((0, 1, []), (2, 4, [(0, 1, 0x3FF)]), (2, 2, [(0, 5, 0x3FF)]), too_long, too_wide):
        out = gram_out(B, 4, 4)
        with pytest.raises(sr_b200.SrError):
            handle.recognise_long_grammar(pcm, g, 1000, 4, 4, 2400, lens, out=out, rate=rate)
        for k, v in out.items():
            assert set(np.asarray(v).tobytes()) <= {CANARY, 0}, (g, k)
    # and the call still works afterwards
    long_pair(handle, pcm, lens, rate, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_digit_recordings(handle, rate):
    lo, port, lg = ox.long_oracle(), ob.port(), ox.long_grammar()
    from cases import digit_bank
    bk, T, K = digit_bank(port, lo, ox.golden_wav(DIGITS[1]))
    handle.set_bank(bk, T, 4096)
    handle.set_match(0, 0)
    xs = [at_rate(ox.golden_wav(n), rate) for n in DIGITS]
    lens = np.array([len(x) for x in xs], np.uint32)
    pcm = np.full((len(xs), int(lens.max())), 2048, np.uint16)
    for b, x in enumerate(xs):
        pcm[b, :len(x)] = x
    got, (y, l8) = long_pair(handle, pcm, lens, rate, 32)
    assert int(got["n_segs"].sum()) > 20
    g = sr_b200.chain_grammar(K, (1 << K) - 1) if K * K <= sr_b200.GRAM_COPY_MAX else LOOP
    gram_pair(handle, pcm, lens, rate, LOOP, 32, 64)
    gram_pair(handle, pcm, lens, rate, g, 32, 64)
    yc, l8c = cpu_eight(pcm[:1], lens[:1], rate)
    assert l8c.tolist() == l8[:1].tolist() and yc[0, :l8c[0]].tobytes() == y[0, :l8c[0]].tobytes()
    want = ox.recognise_long(lo, port, yc, 2400, bk, T, 4096, 32, l8c)
    cmp_long({k: v[:1] for k, v in got.items()}, want, 32)


@pytest.mark.gpu
def test_two_handles_on_two_threads_equal_serial(bank):
    jobs = [(44100, 0x1A80), (16000, 0x1A81)]
    inputs = []
    for rate, seed in jobs:
        U_in, lens = ragged(rate)
        inputs.append((rate, batch_at(rate, lens, seed, U_in), lens))

    def run(h, rate, pcm, lens):
        a = h.recognise_long_batch(pcm, 32, 2400, lens, rate=rate)
        g = h.recognise_long_grammar(pcm, LOOP, 1000, 32, 64, 2400, lens, rate=rate)
        return [np.asarray(v).tobytes() for v in list(a.values()) + list(g.values())]

    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        for h in handles:
            h.set_bank(bank[0], bank[1], 4096)
        serial = [run(h, *x) for h, x in zip(handles, inputs)]
        for rep in range(2):
            out, errors = [None] * len(jobs), []

            def work(i):
                try:
                    out[i] = run(handles[i], *inputs[i])
                except Exception as e:                  # noqa: BLE001
                    errors.append(e)
            th = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert not errors and out == serial, rep
    finally:
        for h in handles:
            h.close()
