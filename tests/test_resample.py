"""sr_resample_adc12_dev (include/sr_synth.h): 12-bit codes at any rate of SR_RESAMPLE_RATES to the 8 kHz codes every other
call takes, checked bit for bit against the numpy restatement in tests/resample_ref.py. CPU tests hold the committed tap
tables to tools/gen_resample_taps.py and to their bounds, and the restatement to its filter's job (a 1 kHz tone passes,
a 5 kHz one does not). GPU tests cover random and full-scale inputs at every rate, edge and ragged lengths, a 30-minute
recording, the bytes the call may write, its refusals, two streams on two threads, and real speech taken up to 16, 44.1
and 48 kHz and brought back before the long-form recogniser. tests/test_concurrency.py enumerates the other headers'
entry points, not sr_synth.h, so the threaded check is here."""
import os
import re
import sys
import threading

import numpy as np
import pytest

import resample_ref as rr
import sr_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_resample_taps as gen  # noqa: E402

CANARY = 0xA5A5
LEN_CANARY = 0x5A5A5A5A


# ---- the tables ---------------------------------------------------------------------------------------------------------
def test_rates_match_the_header_and_binding():
    text = open(os.path.join(ROOT, "include", "sr_synth.h")).read()
    m = re.search(r"#define SR_RESAMPLE_RATES \{([^}]*)\}", text)
    assert tuple(int(v) for v in m.group(1).split(",")) == gen.RATES == sr_b200.RESAMPLE_RATES
    assert "#define SR_RESAMPLE_U_MAX (1u << 30)" in text and sr_b200.RESAMPLE_U_MAX == 1 << 30


def test_committed_taps_equal_generator():
    path = os.path.join(ROOT, "stm32-speech-recognition_b200", "csrc", "sr_resample_taps.h")
    assert open(path).read() == gen.header_text()


def test_tap_counts_and_ratios():
    want = {8000: (1, 1, 1), 11025: (320, 441, 14113), 16000: (1, 2, 65), 22050: (160, 441, 14113),
            32000: (1, 4, 129), 44100: (80, 441, 14113), 48000: (1, 6, 193)}
    for rate in rr.RATES:
        L, M = rr.ratio(rate)
        h = rr.taps(rate)
        assert (L, M, len(h)) == want[rate] and len(h) % 2 == 1
        assert (h == h[::-1]).all()                                    # linear phase: the centre tap is the delay
    assert rr.taps(8000).tolist() == [32768]


def test_every_phase_has_unit_gain_and_exact_s32_sums():
    """per phase: |sum h - 2^15| <= 8 (DC gain within 0.03 %), and 2048 * sum |h| + 2^14 < 2^31, so neither the s32 sum of
    centred codes in [-2048, 2047] nor its rounding add can overflow"""
    for rate in rr.RATES:
        hp = rr.phases(rate)
        assert np.abs(hp.sum(axis=1) - (1 << 15)).max() <= 8, rate
        assert 2048 * np.abs(hp).sum(axis=1).max() + (1 << 14) < 2 ** 31, rate


# ---- the restatement as a filter ----------------------------------------------------------------------------------------
def tone(f, rate, secs=1.0, amp=1500.0):
    t = np.arange(int(rate * secs)) / rate
    return np.rint(2048 + amp * np.sin(2 * np.pi * f * t)).astype(np.uint16)


def rms_db(x):
    """level of the middle half of a code sequence around mid-code (ramps at the ends left out)"""
    v = x.astype(np.float64)[len(x) // 4: 3 * len(x) // 4] - 2048
    return 20 * np.log10(max(np.sqrt((v * v).mean()), 1e-9))


def test_identity_at_8k():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 4096, 10007).astype(np.uint16)
    assert np.array_equal(rr.resample(x, 8000), x)


@pytest.mark.parametrize("rate", rr.RATES)
def test_1khz_tone_keeps_its_level(rate):
    x = tone(1000.0, rate)
    y = rr.resample(x, rate)
    assert len(y) == 8000 and abs(rms_db(y) - rms_db(x)) < 0.1


@pytest.mark.parametrize("rate", [r for r in rr.RATES if r >= 11025])
def test_5khz_tone_is_removed(rate):
    """5 kHz is above the 4 kHz Nyquist of the output; unfiltered it would fold to 3 kHz"""
    x = tone(5000.0, rate)
    assert rms_db(rr.resample(x, rate)) - rms_db(x) <= -60.0


def test_out_len():
    assert rr.out_len(0, 44100) == 0 and rr.out_len(1, 44100) == 1 and rr.out_len(441, 44100) == 80
    assert rr.out_len(442, 44100) == 81 and rr.out_len(7, 48000) == 2 and rr.out_len(6, 48000) == 1


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def run(pcm, rate, lens=None, U_out=None, stream=None, use_lens=True):
    """one call on torch buffers: output rows and out_lens prefilled with canaries; returns (out [B, U_out], out_lens [B])"""
    import torch
    B, U_in = pcm.shape
    L, M = rr.ratio(rate)
    U_out = -(-U_in * L // M) if U_out is None else U_out
    x = _dev(pcm.view(np.int16))
    ln = _dev(np.asarray(lens, np.uint32).view(np.int32)) if (lens is not None and use_lens) else None
    out = torch.full((B, max(U_out, 1)), CANARY - 65536, dtype=torch.int16, device="cuda:0")
    olens = torch.full((max(B, 1),), LEN_CANARY, dtype=torch.int32, device="cuda:0")
    s = torch.cuda.current_stream() if stream is None else stream
    sr_b200.resample_adc12_dev(x.data_ptr(), U_in, B, None if ln is None else ln.data_ptr(), rate, out.data_ptr(), U_out,
                               olens.data_ptr(), s.cuda_stream)
    s.synchronize()
    return out.cpu().numpy().view(np.uint16)[:, :U_out], olens.cpu().numpy().view(np.uint32)[:B]


def check(pcm, rate, lens, U_out=None, **kw):
    got, olens = run(pcm, rate, lens, U_out, **kw)
    lens = np.full(pcm.shape[0], pcm.shape[1]) if lens is None else np.minimum(lens, pcm.shape[1])
    want = rr.resample_batch(pcm, rate, lens, got.shape[1], np.full(got.shape, CANARY, np.uint16))
    assert np.array_equal(olens, [rr.out_len(int(n), rate) for n in lens]), rate
    bad = np.argwhere(got != want)
    assert not len(bad), "rate %d: first difference at %s of %d" % (rate, bad[0], len(bad))
    return got


def edge_lens(rate, U_in):
    """0, 1, 2, around ceil(N / L) (the taps one output meets), around one tile's input, and U_in"""
    L, M = rr.ratio(rate)
    K = -(-len(rr.taps(rate)) // L)
    tile = (2048 if L == 1 else 64 * L) * M // L
    v = [0, 1, 2, K - 1, K, K + 1, 2 * K + 3, tile - 1, tile, tile + 1, U_in - 1, U_in]
    return np.array([n for n in v if 0 <= n <= U_in], np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", rr.RATES)
def test_random_codes_and_edge_lengths(rate):
    rng = np.random.default_rng(rate)
    U_in = 3 * rate // 2 + 17
    lens = np.concatenate([edge_lens(rate, U_in), rng.integers(0, U_in + 1, 12).astype(np.uint32),
                           np.array([U_in + 5, 0xFFFFFFFF], np.uint32)])              # past U_in: read as U_in
    pcm = rng.integers(0, 4096, (len(lens), U_in)).astype(np.uint16)
    U_out = rr.out_len(U_in, rate) + 40                                                # canaries past every row
    check(pcm, rate, lens, U_out)
    check(pcm[:5], rate, None, U_out)                                                  # lens NULL: every row U_in


@pytest.mark.gpu
@pytest.mark.parametrize("rate", rr.RATES)
def test_full_scale_square_waves_hit_both_clamps(rate):
    U_in = rate
    n = np.arange(U_in)
    rows = []
    for period_ms in (1.0, 2.5, 10.0, 31.0):                          # 1 kHz .. 32 Hz, 0 / 4095 codes
        p = max(2, int(rate * period_ms / 1000))
        rows.append(np.where((n % p) < p // 2, 4095, 0))
    rows.append(np.where((n // 3) % 2 == 0, 4095, 0))                # a square near the input's Nyquist
    pcm = np.array(rows, np.uint16)
    got = check(pcm, rate, np.array([U_in, U_in - 1, U_in // 2, 333, U_in], np.uint32))
    assert (got[:3] == 0).any() and (got[:3] == 4095).any(), rate


@pytest.mark.gpu
def test_thirty_minutes_at_48k_on_sampled_windows():
    import torch
    rate, U_in = 48000, 30 * 60 * 48000
    rng = np.random.default_rng(30)
    # a slow random walk with noise on it, so that windows differ and every code range is met
    walk = np.cumsum(rng.integers(-3, 4, U_in // 64 + 1)).repeat(64)[:U_in]
    pcm = np.clip(2048 + (walk % 3000) - 1500 + rng.integers(-400, 401, U_in), 0, 4095).astype(np.uint16)[None]
    U_out = rr.out_len(U_in, rate) + 8
    got, olens = run(pcm, rate, None, U_out)
    n_out = rr.out_len(U_in, rate)
    assert olens[0] == n_out == 14_400_000
    starts = np.concatenate([[0, n_out - 4096], rng.integers(0, n_out - 4096, 30)])
    idx = np.unique(np.concatenate([np.arange(s, s + 4096) for s in starts]))
    assert np.array_equal(got[0, idx], rr.resample(pcm[0], rate, idx))
    assert (got[0, n_out:] == CANARY).all()
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_refusals_write_nothing():
    import torch
    rng = np.random.default_rng(5)
    pcm = rng.integers(0, 4096, (3, 4410)).astype(np.uint16)
    x = _dev(pcm.view(np.int16))
    lens = _dev(np.array([4410, 100, 0], np.int32))
    out = torch.full((3, 1000), CANARY - 65536, dtype=torch.int16, device="cuda:0")
    olens = torch.full((3,), LEN_CANARY, dtype=torch.int32, device="cuda:0")
    host_out = np.full((3, 1000), CANARY, np.uint16)

    def call(rate, U_out, in_ptr=x.data_ptr(), out_ptr=out.data_ptr(), U_in=4410):
        with pytest.raises(sr_b200.SrError):
            sr_b200.resample_adc12_dev(in_ptr, U_in, 3, lens.data_ptr(), rate, out_ptr, U_out, olens.data_ptr())

    for rate in (0, 7999, 8001, 12000, 24000, 96000):
        call(rate, 1000)
    call(44100, rr.out_len(4410, 44100) - 1)                                 # U_out one too small
    call(48000, rr.out_len(4410, 48000) - 1)
    call(44100, 1000, U_in=sr_b200.RESAMPLE_U_MAX + 1)
    call(44100, 1000, in_ptr=0)
    call(44100, 1000, in_ptr=pcm.ctypes.data)                                # host memory
    call(44100, 1000, out_ptr=host_out.ctypes.data)
    call(44100, 1000, in_ptr=x.data_ptr() + 1)                               # misaligned
    torch.cuda.synchronize()
    assert (out.cpu().numpy().view(np.uint16) == CANARY).all() and (host_out == CANARY).all()
    assert (olens.cpu().numpy().view(np.uint32) == LEN_CANARY).all()
    # B = 0 does nothing; U_out exactly the longest out_len is accepted
    sr_b200.resample_adc12_dev(x.data_ptr(), 4410, 0, None, 44100, out.data_ptr(), 800, None)
    sr_b200.resample_adc12_dev(x.data_ptr(), 4410, 3, lens.data_ptr(), 44100, out.data_ptr(), 800, olens.data_ptr())
    torch.cuda.synchronize()
    assert olens.cpu().numpy().tolist() == [800, rr.out_len(100, 44100), 0]


@pytest.mark.gpu
def test_two_streams_on_two_threads_equal_serial():
    import torch
    rng = np.random.default_rng(9)
    jobs = []
    for k, rate in enumerate((44100, 48000, 16000, 11025, 22050, 32000)):
        U_in = rate + 1000 * k
        pcm = rng.integers(0, 4096, (6, U_in)).astype(np.uint16)
        lens = rng.integers(0, U_in + 1, 6).astype(np.uint32)
        jobs.append((pcm, rate, lens))
    serial = [run(p, r, l) for p, r, l in jobs]
    for (p, r, l), (got, _) in zip(jobs[:2], serial[:2]):
        want = rr.resample_batch(p, r, l, got.shape[1], np.full(got.shape, CANARY, np.uint16))
        assert np.array_equal(got, want)
    errors, results = [], {}

    def worker(t):
        try:
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for rep in range(4):
                    for i in range(t, len(jobs), 2):
                        results[(t, rep, i)] = run(*jobs[i], stream=s)
        except Exception as e:                    # pragma: no cover - reported below
            errors.append(repr(e))

    th = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    assert len(results) == 4 * len(jobs)
    for (t, rep, i), (got, ol) in results.items():
        assert np.array_equal(got, serial[i][0]) and np.array_equal(ol, serial[i][1]), (t, rep, i)


# ---- end to end on real speech ------------------------------------------------------------------------------------------
def upsample(x, rate, half=16, beta=8.0):
    """8 kHz codes -> codes at `rate` by a fixed float64 computation: a Kaiser-windowed sinc interpolator with `half`
    input samples a side, cut-off 4 kHz, rounded and clipped to 12 bits"""
    n_out = len(x) * rate // 8000
    pos = np.arange(n_out, dtype=np.float64) * 8000.0 / rate
    base = np.floor(pos).astype(np.int64)
    xc = np.concatenate([np.zeros(half), x.astype(np.float64) - 2048, np.zeros(half + 1)])
    acc = np.zeros(n_out)
    for d in range(-half + 1, half + 1):
        j = base + d
        t = pos - j
        w = np.i0(beta * np.sqrt(np.clip(1 - (t / half) ** 2, 0, None))) / np.i0(beta)
        acc += xc[j + half] * np.sinc(t) * w
    return np.clip(np.rint(acc + 2048), 0, 4095).astype(np.uint16)


# (recording, rate) -> (segments at 8 kHz, segments after the round trip, segments k < both counts whose status and cmd
# equal the 8 kHz run's)
# measured through tests/resample_ref.py and the oracles of the long-form recogniser, which the GPU calls equal bit for bit
E2E_PINNED = {
    ("digits_1_10_b", 16000): (10, 10, 9), ("digits_1_10_b", 44100): (10, 10, 9), ("digits_1_10_b", 48000): (10, 10, 9),
    ("digits_1_10_a", 16000): (10, 3, 0), ("digits_1_10_a", 44100): (10, 3, 1), ("digits_1_10_a", 48000): (10, 3, 0),
    ("digits_1_9_units_b", 16000): (13, 13, 13), ("digits_1_9_units_b", 44100): (13, 13, 13),
    ("digits_1_9_units_b", 48000): (13, 13, 13),
    ("digits_1_9_units_a", 16000): (13, 13, 11), ("digits_1_9_units_a", 44100): (13, 13, 11),
    ("digits_1_9_units_a", 48000): (13, 13, 11),
}


@pytest.mark.gpu
def test_real_speech_round_trip_through_the_long_recogniser():
    """each digit recording's twin enrols the bank (template k = segment k, in slot 4k); the recording itself, taken up
    to 16 / 44.1 / 48 kHz on the CPU and brought back on the GPU, is recognised by sr_recognise_long_batch beside the
    8 kHz original. The segment counts and the number of segments whose decision agrees with the original's are pinned;
    the round trip is not claimed to be transparent beyond those counts."""
    import torch
    import oracle_bind as ob
    import oracle_ext as ox
    from cases import digit_bank, real_speech_pairs
    lo, port = ox.long_oracle(), ob.port()
    h = sr_b200.Handle(0)
    seen = {}
    try:
        for a_name, b_name in real_speech_pairs():
            bank, T, _ = digit_bank(port, lo, ox.golden_wav(a_name))
            h.set_bank(bank, T, 4096)
            b = ox.golden_wav(b_name)
            ref = h.recognise_long_batch(b[None], 32, 2400)
            n_ref = int(ref["n_segs"][0])
            for rate in (16000, 44100, 48000):
                up = upsample(b, rate)
                got, olens = run(up[None], rate)
                back = got[:, :int(olens[0])].copy()
                out = h.recognise_long_batch(back, 32, 2400)
                n = int(out["n_segs"][0])
                m = min(n, n_ref, 32)
                s, r = out["segs"][0, :m], ref["segs"][0, :m]
                agree = int(((s["status"] == r["status"]) & (s["cmd"] == r["cmd"])).sum())
                seen[(b_name, rate)] = (n_ref, n, agree)
    finally:
        h.close()
        torch.cuda.empty_cache()
    print(seen)
    assert seen == E2E_PINNED
