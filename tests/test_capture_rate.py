"""The host-buffer capture calls at any rate of SR_RESAMPLE_RATES (sr_recognise_batch_at_rate,
sr_recognise_batch_multi_at_rate, sr_enrol_batch_at_rate, sr_recognise_connected_batch_at_rate and
sr_recognise_connected_grammar_batch_at_rate, include/sr_synth.h): press-to-talk captures in host memory at 11.025 to
48 kHz, resampled to 8 kHz on the GPU, chunk by chunk for recognise and once per call for the other three.

The definition is an equivalence: the call writes exactly what the 8 kHz call writes on y_b, the U8 = ceil(U_in L / M)
outputs of sr_resample_adc12_dev on each capture. So every GPU test here compares the call with sr_resample_adc12_dev,
a copy back and the 8 kHz host call (both pinned to their oracles elsewhere), byte for byte with canaries around every
output buffer, and a few with the CPU composition tests/resample_ref.py + the oracles.

CPU: the header and the binding, the U_in limit per rate against tests/resample_ref.py, and the chunk rule restated.
GPU: every rate and all five calls (n_len 2400, U8 and one not divisible by 240; atap NULL and in / out; U_in at the
limit and at the calibration edge); the packed transport at 48 kHz (forced plain and packed, odd chunks, codes >= 4096,
a short last chunk); the matchers and both geometries; the enrolment round trip; the loop and a digit-string grammar;
NULL outputs; refusals and B = 0; rate 8000 against the 8 kHz calls; launches and tags; two handles through multi; the
board captures; two handles on two threads."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK_BYTES = 32 << 20             # input PCM per chunk of sr_recognise_batch(_at_rate), csrc/sr_api.cu
TAG_RESAMPLE = 15
RATES = [r for r in rr.RATES if r != 8000]
LOOP = sr_b200.loop_grammar()
DIGIT_STRING = sr_b200.chain_grammar(3, 0x3FF)
CANARY = 0xA5
PAD = 64                           # canary bytes before and after every output buffer
U_LIMIT = {48000: 393210, 44100: 361261, 16000: 131070, 11025: 90315}
FTR = sr_b200.FTR_BYTES
RECOG_BYTES = {"atap": 12, "seg_off": 24, "ftr": FTR, "best_idx": 4, "best_dis": 4, "cmd": 4, "status": 1}
CONN_BYTES = {"atap": 12, "seg_off": 24, "frm_num": 12, "n_words": 4, "total": 8, "status": 1}
CALLS = ("recognise", "enrol", "connected", "grammar")


# ---- the definition, restated ---------------------------------------------------------------------------------------------
def u8(n, rate):
    """ceil(n L / M): the 8 kHz samples of a capture of n input samples"""
    L, M = rr.ratio(rate)
    return -(-n * L // M)


def u_max(rate):
    """the longest capture a call at `rate` takes: U8 <= 65535"""
    L, M = rr.ratio(rate)
    return 65535 * M // L


def chunk_size(U_in, B):
    """captures per chunk of sr_recognise_batch_at_rate: about CHUNK_BYTES of input, a multiple of 8, at least 8"""
    c = CHUNK_BYTES // (2 * U_in)
    c = 8 if c < 8 else c & ~7
    return min(c, B)


def n_chunks(U_in, B):
    return -(-B // chunk_size(U_in, B))


def at_rate(x, rate):
    """8 kHz codes -> codes at `rate` (scipy's polyphase filter), rounded and clipped to 12 bits"""
    L, M = rr.ratio(rate)
    y = resample_poly(np.asarray(x, np.float64) - 2048, M, L)
    return np.clip(np.rint(y + 2048), 0, 4095).astype(np.uint16)


def cal_edge(rate, n_len=2400):
    """the longest capture whose ceil(U_in L / M) is n_len while its floor is n_len - 1"""
    L, M = rr.ratio(rate)
    return -(-n_len * M // L) - 1


def captures_at(rate, B, U_in, seed):
    """B synthetic captures of U_in samples at `rate` (three words each)"""
    x = sr_b200.synth_pcm_host(B, u8(U_in, rate) + 64, seed, 3)
    return np.ascontiguousarray(np.stack([at_rate(x[b], rate)[:U_in] for b in range(B)]))


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_header_and_binding():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sr_synth.h")).read(), flags=re.S)
    commas = {"sr_recognise_batch_at_rate": 6, "sr_recognise_batch_multi_at_rate": 7, "sr_enrol_batch_at_rate": 8,
              "sr_recognise_connected_batch_at_rate": 8, "sr_recognise_connected_grammar_batch_at_rate": 9}
    recog = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "speech_recog.h")).read(), flags=re.S)
    L = sr_b200.lib()
    for name, n in commas.items():
        d = re.search(r"int %s\(([^;]*)\);" % name, text)
        assert d and d.group(1).count(",") == n, name
        assert name not in recog and hasattr(L, name), name
    assert "15 the resampling" in open(os.path.join(ROOT, "include", "speech_recog.h")).read()
    for m in (sr_b200.Handle.recognise, sr_b200.Handle.enrol, sr_b200.Handle.recognise_connected,
              sr_b200.Handle.recognise_connected_grammar, sr_b200.recognise_multi):
        assert inspect.signature(m).parameters["rate"].default is None, m


@pytest.mark.parametrize("rate", RATES)
def test_u_in_limit_matches_resample_ref(rate):
    top = u_max(rate)
    assert u8(top, rate) == rr.out_len(top, rate) <= 65535
    assert u8(top + 1, rate) == rr.out_len(top + 1, rate) == 65536
    if rate in U_LIMIT:
        assert top == U_LIMIT[rate]
    assert u8(cal_edge(rate), rate) == rr.out_len(cal_edge(rate), rate) == 2400
    L, M = rr.ratio(rate)
    assert cal_edge(rate) * L // M == 2399


def test_chunk_rule():
    """the counts the GPU tests below check through the tag-15 records and the transport statistics"""
    assert chunk_size(48000, 1 << 20) == 344 and chunk_size(44100, 1 << 20) == 376 and chunk_size(8000, 1 << 20) == 2096
    assert n_chunks(48000, 1033) == 4 and n_chunks(48000, 1032) == 3
    # by 8 kHz bytes a 48 kHz batch of 1 033 captures would be one chunk
    assert CHUNK_BYTES // (2 * u8(48000, 48000)) & ~7 == 2096
    assert chunk_size(u_max(48000), 1 << 20) == 40 and chunk_size(1, 5) == 5


# ---- the reference: sr_resample_adc12_dev, a copy back, the 8 kHz host call -------------------------------------------------
def gpu_eight(pcm, rate):
    """y [B, U8] from sr_resample_adc12_dev on the rows of pcm"""
    import torch
    B, U_in = pcm.shape
    U8 = u8(U_in, rate)
    x = torch.from_numpy(pcm.view(np.int16)).to("cuda:0")
    out = torch.zeros((B, max(U8, 1)), dtype=torch.int16, device="cuda:0")
    s0 = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U_in, B, None, rate, out.data_ptr(), U8, None, s0.cuda_stream)
    s0.synchronize()
    return np.ascontiguousarray(out.cpu().numpy().view(np.uint16)[:, :U8])


def cpu_eight(pcm, rate):
    B, U_in = pcm.shape
    return rr.resample_batch(pcm, rate, np.full(B, U_in, np.uint32), u8(U_in, rate))


def _bufs(sizes, B, atap_fill=None):
    bufs = {k: np.full(B * n + 2 * PAD, CANARY, np.uint8) for k, n in sizes.items()}
    if atap_fill is not None and "atap" in bufs:
        bufs["atap"][PAD:PAD + B * 12] = atap_fill
    return bufs


def _check_canaries(bufs, sizes, B, null):
    for k, n in sizes.items():
        assert set(bufs[k][:PAD].tobytes()) == {CANARY} and set(bufs[k][PAD + B * n:].tobytes()) == {CANARY}, k
        if k in null:
            assert set(bufs[k][PAD:PAD + B * n].tobytes()) <= {CANARY}, k


def raw(h, call, pcm, rate, n_len=2400, null=(), atap=None, penalty=1000, max_words=6, g=LOOP, slot_stride=4096):
    """one raw call (the 8 kHz call when rate is None) with the outputs named in null passed as NULL, atap prefilled with
    the byte atap (None: atap NULL) and PAD canary bytes before and after every buffer: the buffers, canaries included"""
    B, U = pcm.shape
    L = sr_b200.lib()
    at = () if rate is None else (rate,)
    if call == "recognise":
        sizes = dict(RECOG_BYTES, score=4 * h.n_slot)
    elif call == "enrol":
        sizes = {"bank": slot_stride, "status": 1}
    else:
        sizes = dict(CONN_BYTES, words=24 * max_words)
    nul = set(null) | ({"atap"} if atap is None and "atap" in sizes else set())
    bufs = _bufs(sizes, B, None if "atap" in nul else atap)
    ptr = {k: None if k in nul else bufs[k].ctypes.data + PAD for k in sizes}
    if call == "recognise":
        o = sr_b200.RecogOut(*[ptr[k] for k in sr_b200.RECOG_FIELDS])
        fn = L.sr_recognise_batch if rate is None else L.sr_recognise_batch_at_rate
        rc = fn(h._h, pcm.ctypes.data, U, B, *at, n_len, C.byref(o))
    elif call == "enrol":
        fn = L.sr_enrol_batch if rate is None else L.sr_enrol_batch_at_rate
        rc = fn(h._h, pcm.ctypes.data, U, B, *at, n_len, ptr["bank"], slot_stride, ptr["status"])
    elif call == "connected":
        o = sr_b200.ConnOut(*[ptr[k] for k in sr_b200.CONN_FIELDS])
        fn = L.sr_recognise_connected_batch if rate is None else L.sr_recognise_connected_batch_at_rate
        rc = fn(h._h, pcm.ctypes.data, U, B, *at, n_len, penalty, max_words, C.byref(o))
    else:
        o = sr_b200.ConnOut(*[ptr[k] for k in sr_b200.CONN_FIELDS])
        gr = sr_b200.grammar(g)
        fn = L.sr_recognise_connected_grammar_batch if rate is None else L.sr_recognise_connected_grammar_batch_at_rate
        rc = fn(h._h, pcm.ctypes.data, U, B, *at, n_len, C.byref(gr), penalty, max_words, C.byref(o))
    assert rc == 0, (call, sr_b200.lib().sr_last_error(None))
    _check_canaries(bufs, sizes, B, nul)
    return bufs


def pair(h, call, pcm, rate, y=None, **kw):
    """(the call at `rate`, the composition on y) with the same prefilled outputs: every byte must agree"""
    y = gpu_eight(pcm, rate) if y is None else y
    a = raw(h, call, pcm, rate, **kw)
    b = raw(h, call, y, None, **kw)
    for k in b:
        assert a[k].tobytes() == b[k].tobytes(), (call, rate, k, kw)
    return {k: v[PAD:-PAD] for k, v in a.items()}, y


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bank():
    return ox.synth_bank()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
def test_every_rate_all_calls_equal_composition(handle, bank, rate):
    """all five calls at every rate: n_len 2400, U8 and 1000 (not divisible by 240), atap NULL and in / out, U_in of 1 s,
    at the rate's limit and at the calibration edge"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    pcm = captures_at(rate, 6, rate, 0x2C00 + rate)
    U8 = u8(rate, rate)
    y = gpu_eight(pcm, rate)
    for n_len, atap in ((2400, None), (2400, 0x3C), (U8, None), (1000, 0x3C)):
        for call in CALLS:
            got, _ = pair(handle, call, pcm, rate, y, n_len=n_len, atap=atap)
        if n_len == 1000:                               # atap untouched when n_len % 240 != 0
            assert set(got["atap"].tobytes()) == {0x3C}
    rec, _ = pair(handle, "recognise", pcm, rate, y, atap=0)
    assert (rec["status"] == 0).sum() >= 4
    h2 = sr_b200.Handle(0)
    try:
        h2.set_bank(bank[0], bank[1], 4096)
        m = sr_b200.recognise_multi([handle, h2], pcm, rate=rate, want=sr_b200.RECOG_FIELDS)
        one = handle.recognise(y)
        for k in one:
            assert m[k].tobytes() == one[k].tobytes(), k
    finally:
        h2.close()
    top = u_max(rate)
    big = captures_at(rate, 2, top, 0x2C10 + rate)
    edge = captures_at(rate, 3, cal_edge(rate), 0x2C20 + rate)
    for x in (big, edge):
        yx = gpu_eight(x, rate)
        for call in CALLS:
            pair(handle, call, x, rate, yx, atap=0)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [11025, 44100, 48000])
def test_cpu_oracle_composition(handle, bank, rate):
    """resample_ref, then spch_recg and save_mdl (oracle_bind), the connected and grammar restatements (oracle_ext)"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    pcm = captures_at(rate, 4, rate, 0x2C30 + rate)
    y = cpu_eight(pcm, rate)
    assert gpu_eight(pcm, rate).tobytes() == y.tobytes()
    ora = ob.best_oracle()
    want = ora.recognise_batch(y, 2400, bank[0], bank[1], 4096)
    got = handle.recognise(pcm, rate=rate)
    ok = want["status"] == 0
    assert ok.sum() >= 2 and np.array_equal(got["score"][ok], want["score"][ok])
    for k in ("seg_off", "best_idx", "best_dis", "cmd", "status"):
        assert np.array_equal(got[k].reshape(-1), want[k].reshape(-1)), k
    assert ob.ftr_equal(got["ftr"], want["ftr"])
    slots, st = handle.enrol(pcm, rate=rate)
    e = ob.port().recognise_batch(y, 2400, None, 0, 4096)
    wb = sr_b200.make_bank(e["ftr"])
    wb[e["status"] != 0] = 0xFF
    assert np.array_equal(st, e["status"]) and np.array_equal(slots, wb)
    c = handle.recognise_connected(pcm, 3000, 6, rate=rate)
    cw = ox.recognise_connected(ora, ox.connected(), y, 2400, bank[0], bank[1], 4096, 3000, 6)
    g = handle.recognise_connected_grammar(pcm, DIGIT_STRING, 1000, 6, rate=rate)
    gw = ox.recognise_connected_grammar(ora, ox.grammar(), y, 2400, bank[0], bank[1], 4096, DIGIT_STRING, 1000, 6)
    for got_, want_ in ((c, cw), (g, gw)):
        for k in ("atap", "seg_off", "frm_num", "n_words", "total", "status"):
            assert got_[k].tobytes() == np.asarray(want_[k]).astype(got_[k].dtype).tobytes(), k
        for b in range(len(pcm)):
            n = min(int(got_["n_words"][b]), 6)
            assert got_["words"][b, :n].tobytes() == np.asarray(want_["words"])[b, :n].tobytes(), b


@pytest.mark.gpu
def test_transport_at_48k():
    """>= 4 chunks at 48 kHz, forced plain and forced packed: equal to the composition, packed chunks and input-byte
    H2D counts in transport_stats; an odd U_in with an odd last chunk and a chunk holding a code >= 4096 go plain; the
    last chunk is shorter than the others"""
    h = sr_b200.Handle(0)
    try:
        h.set_bank(*ox.synth_bank(), 4096)
        rate, B = 48000, 4 * 344 + 5
        for U_in, plant in ((48000, False), (48001, False), (48000, True)):
            pcm = np.ascontiguousarray(np.tile(captures_at(rate, 8, U_in, 0x2C40 + U_in), (B // 8 + 1, 1))[:B])
            if plant:
                pcm[3, 100] = 4096                     # chunk 0 holds a code >= 4096
            c = chunk_size(U_in, B)
            assert n_chunks(U_in, B) == 5 and B - 4 * c == 5 < c
            y = gpu_eight(pcm, rate)
            want = h.recognise(y)
            sizes = [min(c, B - i * c) * U_in for i in range(5)]
            for mode in (0, 1):
                h.set_transport(mode)
                got = h.recognise(pcm, rate=rate)
                for k in want:
                    assert got[k].tobytes() == want[k].tobytes(), (U_in, plant, mode, k)
                packed, plain, h2d = h.transport_stats()
                assert packed + plain == 5, (packed, plain)
                if mode == 0:
                    assert packed == 0 and h2d == B * U_in * 2
                    continue
                assert packed >= 1
                if U_in % 2 or plant:
                    assert plain >= 1
                # which chunks went packed is the packers' pace: h2d is one of the sums of 3/2 or 2 bytes per sample
                options = set()
                for mask in range(32):
                    if bin(mask).count("1") == packed:
                        options.add(sum(n // 2 * 3 if (mask >> i) & 1 else n * 2 for i, n in enumerate(sizes)))
                assert h2d in options, (h2d, packed)
    finally:
        h.set_transport(-1)
        h.close()


MATCHERS = [(0, 0), (sr_b200.DTW_BAND, 10), (sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE, 118),
            (sr_b200.DTW_SYM_P1, 10),
            (sr_b200.DTW_BAND | sr_b200.DTW_LIFTER | sr_b200.dtw_knn(3) | sr_b200.dtw_reject(100), 10)]


@pytest.mark.gpu
@pytest.mark.parametrize("geom", (0, 1))
def test_matchers_and_geometry(bank, geom):
    """recognise and multi under every matcher, in both geometries"""
    rate = 44100
    pcm = captures_at(rate, 10, rate, 0x2C50)
    y = gpu_eight(pcm, rate)
    hs = [sr_b200.Handle(0), sr_b200.Handle(0)]
    try:
        for h in hs:
            h.set_bank(bank[0], bank[1], 4096)
            h.set_geometry(geom)
        for flags, r in MATCHERS:
            for h in hs:
                h.set_match(flags, r)
            pair(hs[0], "recognise", pcm, rate, y, atap=0)
            m = sr_b200.recognise_multi(hs, pcm, rate=rate, want=sr_b200.RECOG_FIELDS)
            one = hs[0].recognise(y)
            for k in one:
                assert m[k].tobytes() == one[k].tobytes(), (flags, k)
        pair(hs[0], "enrol", pcm, rate, y)
    finally:
        for h in hs:
            h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100])
def test_enrolment_round_trip(rate):
    """the bank image of sr_enrol_batch_at_rate is sr_enrol_batch's on K15's outputs, and recognising at the rate against
    it equals the composition"""
    h = sr_b200.Handle(0)
    try:
        words = captures_at(rate, 16, rate, 0x2C60 + rate)
        yw = gpu_eight(words, rate)
        slots, st = h.enrol(words, rate=rate)
        s8, st8 = h.enrol(yw)
        assert np.array_equal(slots, s8) and np.array_equal(st, st8) and (st == 0).sum() >= 12
        h.set_bank(slots, len(slots), 4096)
        pcm = np.ascontiguousarray(np.concatenate([words[::2], captures_at(rate, 8, rate, 0x2C70 + rate)]))
        got, _ = pair(h, "recognise", pcm, rate, atap=0)
        assert (got["best_dis"].view(np.uint32)[:8] == 0).sum() >= 6       # the enrolled words find their own slots
        pair(h, "connected", pcm, rate, max_words=8)
    finally:
        h.close()


@pytest.mark.gpu
def test_connected_calls_and_grammars(handle, bank):
    """the loop grammar at a rate equals the connected call at the rate; a digit-string grammar; max_words below the word
    count"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 48000
    pcm = captures_at(rate, 8, 2 * rate, 0x2C80)
    y = gpu_eight(pcm, rate)
    for mw in (1, 2, 16):
        a, _ = pair(handle, "connected", pcm, rate, y, max_words=mw, penalty=3000, atap=0)
        b, _ = pair(handle, "grammar", pcm, rate, y, max_words=mw, penalty=3000, atap=0, g=LOOP)
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), (mw, k)
        if mw == 16:
            assert int(a["n_words"].view(np.uint32).max()) >= 2
        pair(handle, "grammar", pcm, rate, y, max_words=mw, g=DIGIT_STRING)


@pytest.mark.gpu
def test_null_outputs_and_footprint(handle, bank):
    """every output pointer NULL in turn, canaries around every buffer"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 16000
    pcm = captures_at(rate, 5, rate, 0x2C90)
    y = gpu_eight(pcm, rate)
    for call, fields in (("recognise", sr_b200.RECOG_FIELDS), ("connected", sr_b200.CONN_FIELDS),
                         ("grammar", sr_b200.CONN_FIELDS), ("enrol", ("status",))):
        for f in fields:
            pair(handle, call, pcm, rate, y, null=(f,), atap=0)
        pair(handle, call, pcm, rate, y, null=tuple(fields))


@pytest.mark.gpu
def test_refusals_write_nothing_and_b0_launches_nothing(handle, bank):
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 44100
    pcm = captures_at(rate, 3, rate, 0x2CA0)
    over = np.zeros((1, u_max(rate) + 1), np.uint16)
    L = sr_b200.lib()
    cases = [dict(rate=0), dict(rate=7999), dict(rate=12000), dict(rate=96000), dict(pcm=over),
             dict(n_len=u8(rate, rate) + 1), dict(pcm=np.zeros((2, 0), np.uint16))]
    for c in cases:
        x, r, n_len = c.get("pcm", pcm), c.get("rate", rate), c.get("n_len", 2400)
        for call in CALLS:
            sizes = {"recognise": dict(RECOG_BYTES, score=4 * handle.n_slot), "enrol": {"bank": 4096, "status": 1}}.get(
                call, dict(CONN_BYTES, words=24 * 4))
            B = x.shape[0]
            bufs = _bufs(sizes, B)
            p = {k: bufs[k].ctypes.data + PAD for k in sizes}
            l0 = handle.launch_count()
            if call == "recognise":
                rc = L.sr_recognise_batch_at_rate(handle._h, x.ctypes.data, x.shape[1], B, r, n_len,
                                                  C.byref(sr_b200.RecogOut(*[p[k] for k in sr_b200.RECOG_FIELDS])))
            elif call == "enrol":
                rc = L.sr_enrol_batch_at_rate(handle._h, x.ctypes.data, x.shape[1], B, r, n_len, p["bank"], 4096, p["status"])
            elif call == "connected":
                rc = L.sr_recognise_connected_batch_at_rate(handle._h, x.ctypes.data, x.shape[1], B, r, n_len, 1000, 4,
                                                            C.byref(sr_b200.ConnOut(*[p[k] for k in sr_b200.CONN_FIELDS])))
            else:
                rc = L.sr_recognise_connected_grammar_batch_at_rate(
                    handle._h, x.ctypes.data, x.shape[1], B, r, n_len, C.byref(sr_b200.grammar(LOOP)), 1000, 4,
                    C.byref(sr_b200.ConnOut(*[p[k] for k in sr_b200.CONN_FIELDS])))
            assert rc != 0 and handle.launch_count() == l0, (c, call)
            for k in sizes:
                assert set(bufs[k].tobytes()) == {CANARY}, (c, call, k)
        arr = (C.c_void_p * 1)(handle._h)
        rc = L.sr_recognise_batch_multi_at_rate(arr, 1, x.ctypes.data, x.shape[1], x.shape[0], r, n_len,
                                                C.byref(sr_b200.RecogOut(*[None] * 8)))
        assert rc != 0, c
    # what the 8 kHz calls refuse with U8 for U: a bad slot stride, a bank too wide, malformed grammars
    st = np.full(3 + 2 * PAD, CANARY, np.uint8)
    for stride in (2048, 4098):
        assert L.sr_enrol_batch_at_rate(handle._h, pcm.ctypes.data, rate, 3, rate, 2400, st.ctypes.data,
                                        stride, st.ctypes.data + PAD) != 0
    assert set(st.tobytes()) == {CANARY}
    for g in ((0, 1, []), (2, 4, [(0, 1, 0x3FF)]), (2, 2, [(0, 5, 0x3FF)]), sr_b200.chain_grammar(12, 0xFFF)):
        out = {k: np.full(3 * n, CANARY, np.uint8) for k, n in CONN_BYTES.items()}
        with pytest.raises(sr_b200.SrError):
            handle.recognise_connected_grammar(pcm, g, 1000, 4, out=dict(out, words=np.zeros((3, 4), sr_b200.WORD_DTYPE)),
                                               rate=rate)
        for k, v in out.items():
            assert set(v.tobytes()) == {CANARY}, (g, k)
    wide = np.tile(bank[0], (11, 1))[:sr_b200.CONN_SLOT_MAX + 1]
    handle.set_bank(wide, len(wide), 4096)
    for call in ("connected", "grammar"):
        with pytest.raises(AssertionError):
            raw(handle, call, pcm, rate)
    handle.set_bank(bank[0], bank[1], 4096)
    # B = 0 launches nothing, and the call works afterwards
    l0 = handle.launch_count()
    empty = np.zeros((0, rate), np.uint16)
    handle.recognise(empty, rate=rate)
    handle.enrol(empty, rate=rate)
    handle.recognise_connected(empty, 1000, 4, rate=rate)
    handle.recognise_connected_grammar(empty, LOOP, 1000, 4, rate=rate)
    sr_b200.recognise_multi([handle], empty, rate=rate)
    assert handle.launch_count() == l0
    pair(handle, "recognise", pcm, rate, atap=0)


@pytest.mark.gpu
def test_rate_8000_is_the_8khz_call(handle, bank):
    """the same bytes, launch counts, timing tags and transport statistics as the 8 kHz calls, no resample launch"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    pcm = sr_b200.synth_pcm_host(2100 + 5, 8000, 0x2CB0, 3)
    small = np.ascontiguousarray(pcm[:6])
    handle.timing_enable(8192)
    handle.timing_collect()
    runs = []
    for rate in (8000, None):
        c0 = handle.launch_count()
        handle.set_transport(0)
        outs = [handle.recognise(pcm, rate=rate)]
        stats = [handle.transport_stats()]
        outs += [handle.enrol(small, rate=rate), handle.recognise_connected(small, 1000, 8, rate=rate),
                 handle.recognise_connected_grammar(small, LOOP, 1000, 8, rate=rate),
                 sr_b200.recognise_multi([handle], small, rate=rate)]
        runs.append((handle.launch_count() - c0, [t for t, _ in handle.timing_collect()], stats, outs))
    handle.set_transport(-1)
    handle.timing_enable(0)
    (n0, t0, s0, o0), (n1, t1, s1, o1) = runs
    assert n0 == n1 and t0 == t1 and TAG_RESAMPLE not in t0 and s0 == s1
    assert s0[0][1] == 2 and s0[0][2] == pcm.size * 2
    for a, b in zip(o0, o1):
        items = a.items() if isinstance(a, dict) else enumerate(a)
        for k, v in items:
            assert np.asarray(v).tobytes() == np.asarray(b[k]).tobytes(), k


@pytest.mark.gpu
def test_launches_and_tags_at_a_rate(handle, bank):
    """recognise: tag 15 once per chunk, each followed by the 8 kHz call's launches on that chunk; the other three: tag 15
    once, then the 8 kHz call's launches"""
    handle.set_bank(bank[0], bank[1], 4096)
    handle.set_match(0, 0)
    rate = 48000
    B = 2 * 344 + 12
    pcm = np.ascontiguousarray(np.tile(captures_at(rate, 4, rate, 0x2CC0), (B // 4, 1)))
    y = gpu_eight(pcm, rate)
    handle.timing_enable(8192)
    handle.timing_collect()
    handle.set_transport(0)

    def run(f):
        c0 = handle.launch_count()
        f()
        return handle.launch_count() - c0, [t for t, _ in handle.timing_collect()]

    n_rate, t_rate = run(lambda: handle.recognise(pcm, rate=rate))
    n_8k, t_8k = 0, []
    for b0 in range(0, B, 344):
        n, t = run(lambda: handle.recognise(y[b0:b0 + 344]))
        n_8k, t_8k = n_8k + n + 1, t_8k + [TAG_RESAMPLE] + t
    assert n_rate == n_8k and t_rate == t_8k and t_rate.count(TAG_RESAMPLE) == 3
    small, ys = pcm[:6], y[:6]
    for f in (lambda x, r: handle.enrol(x, rate=r), lambda x, r: handle.recognise_connected(x, 1000, 8, rate=r),
              lambda x, r: handle.recognise_connected_grammar(x, LOOP, 1000, 8, rate=r)):
        n_rate, t_rate = run(lambda: f(small, rate))
        n_8k, t_8k = run(lambda: f(ys, None))
        assert n_rate == n_8k + 1 and t_rate == [TAG_RESAMPLE] + t_8k
    handle.set_transport(-1)
    handle.timing_enable(0)


@pytest.mark.gpu
def test_multi_handles_differ_refused(bank):
    hs = [sr_b200.Handle(0), sr_b200.Handle(0)]
    try:
        for h in hs:
            h.set_bank(bank[0], bank[1], 4096)
        hs[1].set_match(sr_b200.DTW_BAND, 10)
        pcm = captures_at(16000, 4, 16000, 0x2CD0)
        with pytest.raises(sr_b200.SrError):
            sr_b200.recognise_multi(hs, pcm, rate=16000)
    finally:
        for h in hs:
            h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_board_captures(handle, bank, rate):
    """the board captures of tests/golden/captures.npz taken to the rate by scipy's resample_poly"""
    cap = np.load(os.path.join(os.path.dirname(__file__), "golden", "captures.npz"))
    xs = [at_rate(cap[k][:16000], rate) for k in sorted(cap.files) if len(cap[k]) >= 16000]
    pcm = np.ascontiguousarray(np.stack(xs))
    slots, st = handle.enrol(np.ascontiguousarray(np.stack([at_rate(cap[k][:8000], rate) for k in sorted(cap.files)])),
                             rate=rate)
    handle.set_bank(slots, len(slots), 4096)
    handle.set_match(0, 0)
    y = gpu_eight(pcm, rate)
    for call in CALLS:
        pair(handle, call, pcm, rate, y, atap=0)
    handle.set_bank(bank[0], bank[1], 4096)


@pytest.mark.gpu
def test_two_handles_on_two_threads_equal_serial(bank):
    jobs = [(44100, 0x2CE0), (16000, 0x2CE1)]
    inputs = [(rate, captures_at(rate, 6, rate, seed)) for rate, seed in jobs]

    def run(h, rate, pcm):
        outs = [h.recognise(pcm, rate=rate), h.enrol(pcm, rate=rate), h.recognise_connected(pcm, 1000, 8, rate=rate),
                h.recognise_connected_grammar(pcm, DIGIT_STRING, 1000, 8, rate=rate)]
        return [np.asarray(v).tobytes() for o in outs for v in (o.values() if isinstance(o, dict) else o)]

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
