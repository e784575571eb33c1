"""GPU parity tests proper: every call goes through the C-ABI of libspeech_b200.so and is compared
BIT-EXACTLY (integer path: tolerance 0) with the oracle -- the reference's own C when oracle/_ref/libref.so
travelled with the repo, else the restatement -- and with the committed golden vectors."""
import ctypes as C
import os

import numpy as np
import pytest

import mfcc_ref as mr
import oracle_bind as ob
import sr_b200
from drive import recognise_dev_np

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CAPS = np.load(os.path.join(HERE, "golden", "captures.npz"))
GOLD = np.load(os.path.join(HERE, "golden", "golden.npz"))


@pytest.fixture(scope="module")
def ora():
    return ob.best_oracle()


def _cmp_recog(out, ref, keys=("seg_off", "score", "best_idx", "best_dis", "cmd", "status")):
    for k in keys:
        assert np.array_equal(out[k].reshape(-1), ref[k].reshape(-1)), k
    assert ob.ftr_equal(out["ftr"], ref["ftr"])


def test_fast_sqrt_exhaustive(handle):
    """the branch-free correctly-rounded sqrt used by mag (MFCC.C:58) and get_dis (DTW.C:59) equals the IEEE
    intrinsic for EVERY float in [1, 2^33) -- a superset of what (float)(s32 pw) and (float)(u32 d) can be"""
    import struct
    lo = struct.unpack("<I", struct.pack("<f", 1.0))[0]
    hi = struct.unpack("<I", struct.pack("<f", 2.0 ** 33))[0]
    bad = C.c_uint64(123)
    rc = sr_b200.lib().sr_debug_sqrt_mismatches(handle._h, lo, hi, C.byref(bad))
    assert rc == 0 and bad.value == 0


# ---- FFT: the asm restatement on device, arbitrary complex inputs -----------------------------------
def test_fft_raw_bit_exact(handle, ora):
    rng = np.random.default_rng(21)
    x = rng.integers(0, 2 ** 32, (96, 1024), dtype=np.uint32)
    x[:4] = 0
    x[4:8] = 0x7FFF7FFF
    x[8:12] = 0x80008000                               # -32768 everywhere: pw = 2^31 corner of MFCC.C:56
    x[12:44, :] = rng.integers(-3000, 3000, (32, 1024)).astype(np.int16).astype(np.uint16)
    assert np.array_equal(handle.fft_raw(x), ora.fft_raw(x))


@pytest.mark.parametrize("length", [0, 1, 160, 161, 256, 1000, 1024])
def test_fft_mag_bit_exact(handle, ora, length):
    rng = np.random.default_rng(length)
    fr = np.ascontiguousarray(rng.integers(-32768, 32768, (16, max(length, 1))).astype(np.int16)[:, :length])
    want = ora.fft_mag(fr) if length else np.zeros((16, 512), np.uint32)      # all-zero input -> all-zero spectrum
    assert np.array_equal(handle.fft_mag(fr), want)


# ---- get_mfcc ----------------------------------------------------------------------------------------
def test_mfcc_fixed_segment_config2_shape(handle, ora):
    """BASELINE config 2 geometry: segment [80, 8000) of every utterance, mid = 2048 -> 98 frames"""
    B, U = 96, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0x5EED0000)
    seg = np.tile(np.array([80, 8000], np.uint32), (B, 1))
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2048
    got = handle.mfcc(pcm, seg, atap)
    assert (got["frm_num"] == 98).all()
    assert ob.ftr_equal(got, ora.mfcc_batch(pcm, seg, atap))


def test_mfcc_extreme_inputs_and_ragged_segments(handle, ora):
    rng = np.random.default_rng(9)
    B, U = 64, 12000
    pcm = rng.integers(0, 4096, (B, U)).astype(np.uint16)
    pcm[:8] = rng.integers(0, 65536, (8, U))           # > 12 bit: s16 window wrap, u32 energy wrap
    pcm[8] = 0
    pcm[9] = 65535
    pcm[10] = 2048                                     # all-zero frames: filter sums 0 -> log(0) pinned to 0
    starts = rng.integers(1, 4000, B) // 1 * 1
    lens = rng.integers(0, 130, B) * 80 + rng.integers(0, 80, B)      # ragged, some < 160, some > 119 frames
    ends = np.minimum(starts + lens, U)
    seg = np.stack([starts, ends], 1).astype(np.uint32)
    seg[11] = [ob.NULL, ob.NULL]
    seg[12] = [100, ob.NULL]
    seg[13] = [80, 80 + 160]                           # exactly one frame
    seg[14] = [80, 80 + 118 * 80 + 160]               # exactly vv_frm_max = 119 frames
    seg[16] = [80, 80 + 119 * 80 + 160]               # 120 frames: rejected, frm_num = 0 (MFCC.C:103-107)
    seg[15] = [1, 1 + 159]                             # one sample short of a frame
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = rng.integers(0, 4096, B)
    atap["mid_val"][10] = 2048                         # row 10 at its own mid_val: every windowed sample and bin is 0
    seg[10] = [100, 100 + 9 * 80 + 160]
    _, sums, _ = mr.mfcc_batch(pcm[10:11], seg[10:11], atap[10:11], mr.GEOM_A)
    assert len(sums) == 10 and (sums == 0).all()
    got = handle.mfcc(pcm, seg, atap)
    valid = (seg[:, 0] != ob.NULL) & (seg[:, 1] != ob.NULL)
    want = ora.mfcc_batch(pcm[valid], seg[valid], atap[valid])
    assert ob.ftr_equal(got[valid], want)
    assert (got["frm_num"][~valid] == 0).all()
    assert (got["frm_num"] == 0).any() and (got["frm_num"] > 100).any() and (got["frm_num"] == 1).any()


@pytest.mark.parametrize("U", [8000, 8003, 5001, 16000])
def test_mfcc_unaligned_utterance_stride(handle, ora, U):
    """utterance strides that break the 16-byte phase of the bulk copies; last utterance ends at the buffer end"""
    B = 37
    pcm = sr_b200.synth_pcm_host(B, U, 0x77 + U)
    rng = np.random.default_rng(U)
    st = rng.integers(1, 900, B)
    en = np.minimum(st + rng.integers(160, 4000, B), U)
    en[-1] = U
    st[0] = 1
    seg = np.stack([st, en], 1).astype(np.uint32)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2000
    assert ob.ftr_equal(handle.mfcc(pcm, seg, atap), ora.mfcc_batch(pcm, seg, atap))


_MFCC_SIZES = [1, 2, 37, 131, 132, 133, 147, 148, 149, 263, 264, 265, 295, 296, 297, 395, 396, 397, 445, 1000]
_MFCC_MIXES = ["rejected_runs", "all_rejected", "all_1", "all_119", "alt_1_119"]


def _mfcc_mix_segments(mix, B, U, rng):
    """segments of one skewed mix; U >= 9839 leaves room for 120-frame segments after a start of up to 79"""
    one, f119, f120 = 160, 118 * 80 + 160, 119 * 80 + 160
    st = rng.integers(1, 80, B)
    if mix == "all_1":
        ln = np.full(B, one)
    elif mix == "all_119":
        ln = np.full(B, f119)
    elif mix == "alt_1_119":
        ln = np.where(np.arange(B) % 2 == 0, one, f119)
    else:
        ln = 160 + 80 * rng.integers(0, 119, B) + rng.integers(0, 80, B)      # 1..119 frames
        rej = np.ones(B, bool)
        if mix == "rejected_runs":                     # 1..3 valid utterances, then 20..30 rejected ones, and so on
            i = 0
            while i < B:
                n_ok = int(rng.integers(1, 4))
                rej[i:i + n_ok] = False
                i += n_ok + int(rng.integers(20, 31))
        kind = np.arange(B) % 3                        # rejected: 120 frames (MFCC.C:103-107), < one frame, NULL
        ln = np.where(rej & (kind == 0), f120 + rng.integers(0, 80, B), ln)
        ln = np.where(rej & (kind == 1), rng.integers(0, 160, B), ln)
    seg = np.stack([st, st + ln], 1).astype(np.uint32)
    if mix in ("rejected_runs", "all_rejected"):
        seg[rej & (kind == 2)] = [ob.NULL, ob.NULL]
        assert rej.sum() >= min(B, 20) or (mix == "rejected_runs" and B <= 3)     # a run starts with 1..3 valid ones
    assert (seg[seg[:, 1] != ob.NULL, 1] <= U).all()
    return seg


@pytest.mark.parametrize("B,mix", [pytest.param(B, "ragged", id=str(B)) for B in _MFCC_SIZES] +
                         [pytest.param(B, m, id="%s-%d" % (m, B)) for m in _MFCC_MIXES for B in _MFCC_SIZES])
def test_mfcc_batch_sizes_around_the_cta_count(handle, ora, B, mix):
    """mfcc_kernel hands utterances out with an atomic counter and ends a CTA's walk with an end marker in its staging
    ring; batch sizes around 1x / 2x / 3x the CTA count make every mix of (utterance, marker) land in a CTA's first
    ring slots, in either claim order (the first version lost an utterance that sat behind a marker); 132 is the H100's
    CTA count. The mixes skew the work per ring slot: a rejected utterance (F = 0) passes the ring without a frame loop,
    yet every consumer warp must still arrive on its `empty` barrier; runs of 20+ of them, all rejected, all 1 frame, all
    119 frames, 1 / 119 alternating. Run twice: the last CTA out re-arms the counter for the next launch; an all-NULL
    launch in between overwrites every frm_num, so an utterance the second launch lost cannot show the first launch's rows."""
    if mix == "ragged":
        U = 4003
        pcm = sr_b200.synth_pcm_host(B, U, 0x4A00 + B)
        rng = np.random.default_rng(B)
        st = rng.integers(1, 900, B)
        en = np.minimum(st + rng.integers(160, 3000, B), U)
        seg = np.stack([st, en], 1).astype(np.uint32)
    else:
        U = 9843
        pcm = sr_b200.synth_pcm_host(B, U, 0x4B00 + B, 2)
        seg = _mfcc_mix_segments(mix, B, U, np.random.default_rng(0x4B00 + B))
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2000
    valid = (seg != ob.NULL).all(axis=1)
    want = ora.mfcc_batch(pcm[valid], seg[valid], atap[valid])
    if mix == "all_rejected":
        assert (want["frm_num"] == 0).all()
    elif mix != "ragged":
        assert (want["frm_num"] > 0).any()
    nulls = np.full((B, 2), ob.NULL, np.uint32)
    for _ in range(2):
        got = handle.mfcc(pcm, seg, atap)
        assert ob.ftr_equal(got[valid], want) and (got["frm_num"][~valid] == 0).all()
        assert (handle.mfcc(pcm, nulls, atap)["frm_num"] == 0).all()


def test_mfcc_segment_at_sample_zero_pins_mid_val(handle, ora):
    """start == 0 makes MFCC.C:119 read vc_dat[-1], which is not a sample of the utterance (the last sample of row b-1,
    or before the batch). The batched forms pin it to the utterance's own mid_val in every row: the features equal the
    oracle on [mid_val, row...]. The rows before are made to end far from mid (0 / 4095), and the start-0 segments sit at
    every 16-byte phase of the bulk copy (U = 4003) and, through device pointers 2, 6 and 14 bytes past a 16-byte
    boundary, in the cooperative copy. Segments that start at 1 read their own sample 0."""
    for U in (4000, 4003):
        _check_sample_zero_pins_mid_val(handle, ora, U)


def _check_sample_zero_pins_mid_val(handle, ora, U):
    import torch
    B = 11
    pcm = sr_b200.synth_pcm_host(B, U, 0x99)
    pcm[:, -1] = np.where(np.arange(B) % 2 == 0, 0, 4095)
    seg = np.tile(np.array([0, 1600], np.uint32), (B, 1))
    seg[3] = (0, U)
    seg[5] = (1, 1601)
    seg[6] = (0, 159)                                  # less than a frame
    seg[8] = (0, 160)                                  # exactly one frame
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2100
    atap["mid_val"][4] = 300
    want = ora.mfcc_batch(ob.pinned_rows(pcm, atap), seg + 1, atap)
    assert want["frm_num"][6] == 0 and want["frm_num"][8] == 1 and want["frm_num"][3] == (U - 160) // 80 + 1
    assert ob.ftr_equal(handle.mfcc(pcm, seg, atap), want), U
    dev = torch.device("cuda:0")
    h = sr_b200.Handle(0)
    st = torch.cuda.Stream(dev)
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        buf = torch.zeros(B * U + 16, dtype=torch.int16, device=dev)
        seg_d, atm_d = _to_dev(seg), _to_dev(atap)
        for k in (0, 1, 3, 7):                         # 0: aligned base (bulk copy); else 2k bytes past a boundary
            buf.fill_(4095)
            buf[k:k + B * U] = torch.from_numpy(pcm.view(np.int16).reshape(-1)).to(dev)
            ptr = buf.data_ptr() + 2 * k
            assert (ptr % 16 == 0) == (k == 0)
            ft = torch.full((B * sr_b200.FTR_BYTES,), 0x5A, dtype=torch.uint8, device=dev)
            h.mfcc_dev(ptr, U, B, seg_d.data_ptr(), 2, atm_d.data_ptr(), ft.data_ptr())
            st.synchronize()
            assert ob.ftr_equal(ft.cpu().numpy().view(sr_b200.FTR_DTYPE), want), (U, k)
    h.close()


def _windowed(x, prv, mid, hamm):
    """vc_temp of MFCC.C:118-121 in the C types: (x - mid) - (prv - mid)*95/100 in s32 with truncating division, times
    hamm[i], / 1000 truncating, cast to s16 (no intermediate here leaves s32)"""
    def cdiv(a, d):                                        # C division: truncates toward zero
        return np.sign(a) * (np.abs(a) // d)
    cur, p = x.astype(np.int64) - mid, prv.astype(np.int64) - mid
    t = cur - cdiv(p * 95, 100)
    return cdiv(t * hamm, 1000).astype(np.int16)


def _full_scale_frames(targets, mids, prv0, hamm):
    """one 160-sample frame per row of `targets`: sample n is the u16 (0..65535) whose windowed value is closest to
    targets[:, n], given the sample chosen before it (prv0 for n = 0)"""
    cand = np.arange(65536, dtype=np.int64)[None, :]
    mid = np.asarray(mids, np.int64)[:, None]
    prv = np.asarray(prv0, np.int64)[:, None]
    out = np.zeros(targets.shape, np.uint16)
    for n in range(160):
        w = _windowed(cand, prv, mid, int(hamm[n])).astype(np.int64)
        out[:, n] = np.argmin(np.abs(w - targets[:, n:n + 1]), axis=1)
        prv = out[:, n:n + 1].astype(np.int64)
    return out


def test_mfcc_largest_magnitude_frames(handle, ora):
    """one-frame segments whose windowed samples sit at +-full scale: constants, the +-alternation, and
    +-32767*sign(cos(2 pi k n / 1024 + phi)) for a spread of bins k. They reach the largest stage-0 values (+-8192) and
    final FFT components near the bound 160*32768/1024 = 5120 that the pruned FFT's no-wrap proof (sr_mfcc.cu header)
    rests on -- synthetic speech and random PCM stay far below it"""
    hamm = np.load(os.path.join(HERE, "golden", "ref_tables.npz"))["hamm"].astype(np.int64)
    n = np.arange(160)
    tg = [np.full(160, 32767), np.full(160, -32768), np.where(n % 2 == 0, 32767, -32768), np.where(n % 2 == 0, -32768, 32767)]
    for k in (0, 1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 144, 233, 256, 377, 448, 500, 511):
        for phi in (0.0, np.pi / 3):
            tg.append(np.where(np.cos(2 * np.pi * k * n / 1024 + phi) >= 0, 32767, -32768))
    targets = np.stack(tg).astype(np.int64)
    B, U = targets.shape[0], 173
    rng = np.random.default_rng(5120)
    mids = rng.choice([0, 2048, 32768, 65535], B)
    mids[:4] = 2048
    prv0 = rng.integers(0, 65536, B)
    frames = _full_scale_frames(targets, mids, prv0, hamm)
    pcm = rng.integers(0, 65536, (B, U)).astype(np.uint16)
    pcm[:, 2] = prv0                                       # x[-1] of the segment [3, 163)
    pcm[:, 3:163] = frames
    seg = np.tile(np.array([3, 163], np.uint32), (B, 1))
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = mids
    # the frames reach what they are built for, on the oracle's FFT of the same windowed samples
    w = np.stack([_windowed(pcm[b, 3:163], pcm[b, 2:162], int(mids[b]), hamm) for b in range(B)])
    assert (np.abs(w.astype(np.int64)) >= 32000).mean() > 0.9
    st0 = w.astype(np.int32) >> 2                          # stage 0 of a real frame: w >> 2
    assert (st0 == -8192).any() and (st0 == 8191).any()
    packed = np.zeros((B, 1024), np.uint32)
    packed[:, :160] = w.view(np.uint16)
    raw = ora.fft_raw(packed)
    comp = np.maximum(np.abs(raw.view(np.int16)[:, 0::2].astype(np.int32)), np.abs(raw.view(np.int16)[:, 1::2].astype(np.int32)))
    assert 0.9 * 5120 <= comp.max() <= 8209
    assert np.array_equal(handle.fft_raw(packed), raw)
    got = handle.mfcc(pcm, seg, atap)
    assert (got["frm_num"] == 1).all()
    assert ob.ftr_equal(got, ora.mfcc_batch(pcm, seg, atap))


# ---- noise_atap + VAD ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["stm32_123", "stm32_456", "stm32_noise", "stm32_voice_123", "v1"])
def test_vad_on_board_captures_matches_golden(handle, name):
    pcm = CAPS[name].reshape(1, -1)
    atap = handle.noise_atap(pcm, 2400)
    assert atap.tobytes() == GOLD[name + "/atap"].tobytes()
    seg = handle.vad(pcm, atap)
    assert seg.reshape(-1).tolist() == GOLD[name + "/seg"].tolist()


def test_vad_extremes_bit_exact(handle, ora):
    rng = np.random.default_rng(4)
    B, U = 48, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0xABCD0000)
    pcm[0] = rng.integers(0, 4096, U)
    pcm[1] = rng.integers(0, 65536, U)
    pcm[2] = 2048
    pcm[3, 2400:] = np.where(np.arange(U - 2400) % 2 == 0, 0, 4095)
    pcm[4, 3000:7900] = rng.integers(0, 4096, 4900)
    for b in range(5, 16):                            # sparse out-of-band spikes: exercises the carried last_sig
        pcm[b] = 2048 + rng.integers(-3, 4, U)
        idx = rng.integers(2400, U, 60)
        pcm[b, idx] = np.where(rng.integers(0, 2, 60) == 1, 2048 + 500, 2048 - 500)
    atap = handle.noise_atap(pcm, 2400)
    seg = handle.vad(pcm, atap)
    for b in range(B):
        a = ora.noise_atap(pcm[b], 2400)
        assert a.tobytes() == atap[b:b + 1].tobytes(), b
        assert ora.vad(pcm[b], U, a).tolist() == seg[b].reshape(-1).tolist(), b
    # n_len not a multiple of 240 leaves atap untouched (VAD.C:33-36)
    keep = atap.copy()
    keep["mid_val"] = 7
    assert handle.noise_atap(pcm, 2401, keep.copy()).tobytes() == keep.tobytes()


@pytest.mark.parametrize("U,buf_len", [(8000, 8000), (8000, 7777), (16000, 16000), (40000, 40000), (8003, 8003), (400, 400), (160, 160)])
def test_vad_lengths(handle, ora, U, buf_len):
    B = 9
    pcm = sr_b200.synth_pcm_host(B, U, 0x1234 + U, 3 if U > 20000 else 1)
    n_len = 2400 if U >= 2400 else (240 if U >= 240 else 0)    # n_len = 0: noise_atap leaves atap untouched
    atap0 = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap0["mid_val"], atap0["n_thl"], atap0["z_thl"], atap0["s_thl"] = 2000, 40, 2, 3000
    atap = handle.noise_atap(pcm, n_len, atap0.copy())
    seg = handle.vad(pcm, atap, buf_len)
    for b in range(B):
        a = ora.noise_atap(pcm[b], n_len, atap0[b:b + 1]) if n_len else atap0[b:b + 1].copy()
        assert a.tobytes() == atap[b:b + 1].tobytes()
        if buf_len > 160:
            assert ora.vad(pcm[b], buf_len, a).tolist() == seg[b].reshape(-1).tolist(), b
        else:
            assert (seg[b] == ob.NULL).all()


def test_noise_atap_windows_longer_than_one_chunk(handle, ora):
    """noise windows beyond the 2 560 samples the kernel stages per chunk take the direct global-memory path"""
    B, U = 40, 16000
    pcm = sr_b200.synth_pcm_host(B, U, 0x5150)
    for n_len in (2640, 4800, 7200, 15840):
        atap = handle.noise_atap(pcm, n_len)
        seg = handle.vad(pcm, atap)
        for b in range(B):
            a = ora.noise_atap(pcm[b], n_len)
            assert a.tobytes() == atap[b:b + 1].tobytes(), (n_len, b)
            assert ora.vad(pcm[b], U, a).tolist() == seg[b].reshape(-1).tolist(), (n_len, b)


def _first_bad_rows(got, want):
    return np.nonzero((got != want).reshape(got.shape[0], -1).any(axis=1))[0][:8].tolist()


@pytest.mark.parametrize("U,sized_for", [(8000, "vad"), (16000, "vad"), (40000, "vad"), (65535, "vad"), (16000, "noise_atap")])
def test_vad_handout_around_sms_times_warps(ora, U, sized_for):
    """vad_kernel: one CTA per SM, one warp per utterance, the next utterance claimed early from an atomic counter that
    the last warp out re-arms. Batch sizes n*W - 1, n*W, n*W + 1 (n = 1, 2) for W = SMs x warps per CTA, where the warps
    per CTA shrink with U (20 at 8 000 and for noise_atap alone, 18 at 16 000, 15 at 40 000, 13 at 65 535): noise_atap
    then VAD, each launched twice on the same handle into outputs refilled with a sentinel, against the oracle"""
    import torch
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def warps_per_cta(buf_len):                        # the formula of launch_vad (sr_vad.cu); noise_atap alone: buf_len 0
        max_frames = 2 * ((((buf_len - 160 + 79) // 80) if buf_len > 160 else 0) + 2)
        per_warp = 2 * (2560 * 2 + 32) + max_frames * 4
        return min(220 * 1024 // per_warp, 20)

    W = sms * warps_per_cta(U if sized_for == "vad" else 0)
    assert warps_per_cta(0) == 20 and warps_per_cta(U) == {8000: 20, 16000: 18, 40000: 15, 65535: 13}[U]
    sizes = [n * W + d for n in (1, 2) for d in (-1, 0, 1)]
    Bmax = sizes[-1]
    pcm = sr_b200.synth_pcm_host(Bmax, U, 0x7AD00000 + U, max(1, (U - 3200) // 5000))
    rng = np.random.default_rng(U)
    for r in (0, W - 1, W, 2 * W):
        pcm[r] = 2048                                  # silence: no segment
    for r in (1, W + 1, 2 * W - 1):
        pcm[r] = rng.integers(0, 65536, U)             # full range
    want_a = np.concatenate([ora.noise_atap(pcm[b], 2400) for b in range(Bmax)])
    want_s = np.stack([ora.vad(pcm[b], U, want_a[b:b + 1]) for b in range(Bmax)])
    assert (want_s[:, 1] != ob.NULL).mean() > 0.9
    h = sr_b200.Handle(0)
    st = torch.cuda.Stream(dev)
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        pcm_d = torch.from_numpy(pcm.view(np.int16)).to(dev)
        at = torch.empty(Bmax * 12, dtype=torch.uint8, device=dev)
        sg = torch.empty(Bmax * 6, dtype=torch.int32, device=dev)
        for B in sizes:
            for run in range(2):
                at.fill_(0xA5 + run)
                sg.fill_(0x5A5A5A5A + run)
                h.noise_atap_dev(pcm_d.data_ptr(), U, B, 2400, at.data_ptr())
                h.vad_dev(pcm_d.data_ptr(), U, B, U, at.data_ptr(), sg.data_ptr())
                st.synchronize()
                got_a = at.cpu().numpy()
                got_s = sg.cpu().numpy().view(np.uint32).reshape(Bmax, 6)
                assert (got_a[B * 12:] == 0xA5 + run).all() and (got_s[B:] == 0x5A5A5A5A + run).all(), (B, run)
                ga = got_a[:B * 12].view(np.uint8).reshape(B, 12)
                assert np.array_equal(ga, want_a[:B].view(np.uint8).reshape(B, 12)), (B, run, _first_bad_rows(ga, want_a[:B].view(np.uint8).reshape(B, 12)))
                assert np.array_equal(got_s[:B], want_s[:B]), (B, run, _first_bad_rows(got_s[:B], want_s[:B]))
    h.close()


def test_vad_and_mfcc_fuzz_with_arbitrary_atap(handle, ora):
    """random PCM shapes and ARBITRARY adaptive parameters handed straight to VAD / get_mfcc (n_thl > mid makes the lower
    band edge wrap, VAD.C:113; huge mid_val exercises the s32 casts of MFCC.C:110,119)"""
    rng = np.random.default_rng(77)
    B, U = 256, 4000
    pcm = np.zeros((B, U), np.uint16)
    for b in range(B):
        kind = b % 6
        base = int(rng.integers(0, 4096))
        if kind == 0:
            pcm[b] = rng.integers(0, 4096, U)
        elif kind == 1:
            pcm[b] = np.clip(base + rng.integers(-30, 31, U), 0, 65535)
            idx = rng.integers(0, U, 200)
            pcm[b, idx] = rng.integers(0, 4096, 200)
        elif kind == 2:
            t = np.arange(U)
            pcm[b] = np.clip(2048 + 1500 * np.sin(t * rng.uniform(0.01, 1.5)) * (rng.random(U) < 0.7), 0, 4095)
        elif kind == 3:
            pcm[b] = rng.integers(0, 65536, U)
        elif kind == 4:
            pcm[b] = np.where(rng.random(U) < 0.05, rng.integers(0, 4096, U), base)
        else:
            blocks = rng.integers(0, 2, U // 80 + 1).repeat(80)[:U]
            pcm[b] = np.where(blocks == 1, rng.integers(0, 4096, U), base)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = rng.integers(0, 4096, B)
    atap["n_thl"] = rng.integers(0, 3000, B)          # often > mid_val: b_thl wraps
    atap["z_thl"] = rng.integers(0, 12, B)
    atap["s_thl"] = rng.integers(0, 200000, B)
    atap["mid_val"][:8] = rng.integers(60000, 2 ** 32, 8, dtype=np.uint64).astype(np.uint32)
    seg = handle.vad(pcm, atap)
    for b in range(B):
        assert ora.vad(pcm[b], U, atap[b:b + 1]).tolist() == seg[b].reshape(-1).tolist(), b
    st = rng.integers(1, 2000, B)
    en = np.minimum(st + rng.integers(160, 1800, B), U)
    sg = np.stack([st, en], 1).astype(np.uint32)
    assert ob.ftr_equal(handle.mfcc(pcm, sg, atap), ora.mfcc_batch(pcm, sg, atap))


def test_vad_threshold_corner_cases(handle, ora):
    """band edges at the corners of the packed 16-bit compare path: a_thl == 0, a_thl > 0xFFFF, b_thl == 0, b_thl wrapped
    (VAD.C:112-113 are u32), mid_val beyond the sample range, thresholds equal to sample values; full-range u16 samples"""
    rng = np.random.default_rng(2024)
    combos = [(0, 0), (0, 1), (1, 1), (5, 5), (5, 6), (100, 100), (2048, 0), (2048, 2048), (2048, 2049), (65535, 0),
              (65535, 1), (65000, 535), (65000, 536), (65000, 2000), (65535, 65535), (30000, 30000), (30000, 40000),
              (65536, 1), (65536, 65535), (70000, 5000), (70000, 4464), (70000, 4465), (2 ** 32 - 5, 10), (2 ** 32 - 1, 0),
              (2 ** 32 - 1, 1), (2 ** 31, 65535), (1, 0), (1, 2), (32768, 32768), (32768, 32767)]
    B, U = len(combos) * 3, 4000
    pcm = np.zeros((B, U), np.uint16)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    for i, (mid, n) in enumerate(combos * 3):
        kind = i // len(combos)
        centre = min(mid, 65535)
        if kind == 0:
            pcm[i] = rng.integers(0, 65536, U)
        elif kind == 1:                                  # hover around the band edges so >=, < and == all occur
            pcm[i] = np.clip(centre + rng.integers(-3, 4, U) + rng.choice([-n, 0, n], U), 0, 65535)
        else:                                            # sparse excursions: long in-band runs between markers
            pcm[i] = centre
            idx = rng.integers(0, U, 120)
            pcm[i, idx] = rng.choice([0, 65535, max(centre - n, 0), min(centre + n, 65535), max(centre - n - 1, 0)], 120)
        atap[i] = (mid, n, int(rng.integers(0, 6)), int(rng.integers(0, 400000)))
    seg = handle.vad(pcm, atap)
    for b in range(B):
        assert ora.vad(pcm[b], U, atap[b:b + 1]).tolist() == seg[b].reshape(-1).tolist(), (b, combos[b % len(combos)])


def test_dtw_limit_batch_and_drop_in_symbol(handle, ora):
    """dtw_limit (DTW.C:76-109): every lattice point of a few (I, M) shapes, and the reference-named symbol after dtw()"""
    L = sr_b200.lib()
    pts = []
    for (I, M) in ((36, 34), (50, 100), (100, 50), (119, 60), (1, 1), (8, 15)):
        for x in range(0, I + 3):
            for y in range(0, M + 3):
                pts.append((x, y, I, M))
    a = np.array(pts, np.uint16)
    out = np.zeros(len(pts), np.uint8)
    cols = [np.ascontiguousarray(a[:, k]) for k in range(4)]
    rc = L.sr_dtw_limit_batch(handle._h, *[c.ctypes.data_as(C.c_void_p) for c in cols], len(pts), out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    po = ob.port()
    want = np.array([po.lib.sro_dtw_limit(int(x), int(y), int(I), int(M)) for x, y, I, M in pts], np.uint8)
    assert np.array_equal(out, want) and 0 < want.sum() < len(pts)
    f = sr_b200.synth_ftr_host(2, 0xABC, 30, 40).view(sr_b200.FTR_DTYPE).reshape(-1)
    L.dtw(f[0:1].ctypes.data_as(C.c_void_p), f[1:2].ctypes.data_as(C.c_void_p))
    I, M = int(f["frm_num"][0]), int(f["frm_num"][1])
    for x, y in ((1, 1), (5, 20), (20, 5), (I, M), (2, 9)):
        assert L.dtw_limit(x, y) == po.lib.sro_dtw_limit(x, y, I, M)
    # ... and against the reference's OWN dtw_limit, which reads the file statics its dtw() left behind (DTW.C:65-68,
    # 130-131, 141-142): call dtw() in libref, then compare every lattice point of that shape with the drop-in symbol
    if ob.have_ref():
        r = ob.ref()
        for seed, lo, hi in ((0xABC, 30, 40), (0x51, 50, 100), (0x52, 8, 15), (0x53, 100, 119)):
            f = sr_b200.synth_ftr_host(2, seed, lo, hi).view(sr_b200.FTR_DTYPE).reshape(-1)
            if seed == 0x51:
                f["frm_num"][0], f["frm_num"][1] = 50, 100        # the 2:1 edge of the guard (DTW.C:133)
            pa, pb = f[0:1].ctypes.data_as(C.c_void_p), f[1:2].ctypes.data_as(C.c_void_p)
            assert L.dtw(pa, pb) == r.lib.dtw(pa, pb)
            I, M = int(f["frm_num"][0]), int(f["frm_num"][1])
            mine = [L.dtw_limit(x, y) for x in range(0, I + 3) for y in range(0, M + 3)]
            theirs = [r.lib.dtw_limit(C.c_uint16(x), C.c_uint16(y)) for x in range(0, I + 3) for y in range(0, M + 3)]
            assert mine == theirs and 0 < sum(theirs) < len(theirs), (seed, I, M)


def test_dtw_fuzz_many_pairs(handle, ora):
    """20 000 random pairs over all length combinations, realistic and adversarial value ranges, T not a multiple of 32"""
    rng = np.random.default_rng(78)
    B, T = 400, 50
    ftr = sr_b200.synth_ftr_host(B, 0xF00D, 1, 119).view(sr_b200.FTR_DTYPE).reshape(-1).copy()
    ftr["mfcc_dat"][::3] = rng.integers(-32768, 32768, ftr["mfcc_dat"][::3].shape)      # every third: full-range values
    ftr["mfcc_dat"][1::7] //= 64                                                          # small values: many equal distances (ties)
    bank = sr_b200.synth_ftr_host(T, 0xFEED, 1, 119, stride=2860)
    bank[::5, 4:] = rng.integers(0, 256, bank[::5, 4:].shape)
    handle.set_bank(bank, T, 2860)
    want, _ = ora.dtw_batch(ftr, bank, T, 2860)
    score, bi, bd = handle.dtw(ftr)
    assert np.array_equal(score, want)


# ---- dtw ---------------------------------------------------------------------------------------------
def test_dtw_all_lengths_bit_exact(handle, ora):
    B, T = 150, 70
    ftr = sr_b200.synth_ftr_host(B, 0xD7A00000, 1, 119).view(sr_b200.FTR_DTYPE).reshape(-1)
    bank = sr_b200.synth_ftr_host(T, 0xD7A10000, 1, 119, stride=4096)
    bank[5, 0] = 0                                     # save_sign != 12345
    bank[17, :2] = 0xFF
    handle.set_bank(bank, T, 4096)
    want, _ = ora.dtw_batch(ftr, bank, T, 4096, check_sign=0)
    score, bi, bd = handle.dtw(ftr, flags=0)
    assert np.array_equal(score, want)
    key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
    k = key.min(axis=1)
    assert np.array_equal(bi, (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)) and np.array_equal(bd, (k >> np.uint64(32)).astype(np.uint32))
    want_s, _ = ora.dtw_batch(ftr, bank, T, 4096, check_sign=1)
    score_s, _, _ = handle.dtw(ftr, flags=sr_b200.DTW_CHECK_SIGN)
    assert np.array_equal(score_s, want_s) and (score_s[:, 5] == ob.NULL).all()


def test_dtw_200_templates_mixed_save_sign(handle, ora):
    """configs[2] bank width: T = 200 = 6 full template tiles + a remainder launch, a third of the slots erased / unsigned
    (main.c:283), against the reference's own dtw; argmin = strict '<' first-wins scan over the 200 slots (main.c:285-289)"""
    B, T = 96, 200
    fin = sr_b200.synth_ftr_host(B, 0xD7A00000, 50, 100).view(sr_b200.FTR_DTYPE).reshape(-1)
    bank = sr_b200.synth_ftr_host(T, 0xD7A10000, 50, 100, stride=4096)
    rng = np.random.default_rng(200)
    bad = rng.random(T) < 0.33
    bank[bad, 0:2] = 0xFF                                  # erased flash: save_sign != 12345
    bank[~bad, 0], bank[~bad, 1] = 12345 & 0xFF, 12345 >> 8
    bank[7] = bank[3]                                      # an exact duplicate: first wins
    handle.set_bank(bank, T, 4096)
    score, bi, bd = handle.dtw(fin, flags=sr_b200.DTW_CHECK_SIGN)
    want, _ = ora.dtw_batch(fin, bank, T, 4096, check_sign=1)
    assert np.array_equal(score, want)
    assert (score[:, bad] == ob.NULL).all() and (score[:, ~bad] != ob.NULL).any()
    key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
    k = key.min(axis=1)
    assert np.array_equal(bi, (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)) and np.array_equal(bd, (k >> np.uint64(32)).astype(np.uint32))
    # same bank without the save_sign check (dtw() itself never looks at it)
    score2, _, _ = handle.dtw(fin)
    want2, _ = ora.dtw_batch(fin, bank, T, 4096, check_sign=0)
    assert np.array_equal(score2, want2)


def test_dtw_empty_feature_sets_are_deterministic(handle, ora):
    """frm_num == 0 on both sides passes the 2:1 guard (DTW.C:133) and the do-while still reads rows 0 and 1 of both
    structs (DTW.C:146-160): the result is defined by the struct bytes, not by whatever was staged before"""
    f = sr_b200.synth_ftr_host(6, 0xE0, 20, 30).view(sr_b200.FTR_DTYPE).reshape(-1).copy()
    f["frm_num"][:3] = 0                                   # rows stay: the reference reads them
    bank = np.zeros((4, 4096), np.uint8)
    bank[:, :2860] = f[[0, 1, 3, 4]].view(np.uint8).reshape(4, 2860)
    handle.set_bank(bank, 4, 4096)
    for _ in range(2):                                     # twice: the second run sees different leftovers in shared memory
        score, _, _ = handle.dtw(f)
        want, _ = ora.dtw_batch(f, bank, 4, 4096)
        assert np.array_equal(score, want)
        handle.dtw(sr_b200.synth_ftr_host(64, 0xE1, 90, 119).view(sr_b200.FTR_DTYPE).reshape(-1))


@pytest.mark.parametrize("T,B,fr", [(1, 70, (1, 119)), (5, 333, (20, 45)), (20, 1500, (23, 43)), (32, 257, (50, 100)),
                                    (33, 640, (1, 119)), (70, 200, (30, 119)), (200, 300, (50, 100))])
def test_dtw_dynamic_pair_scheduling_equals_static_and_reference(ora, T, B, fr):
    """sr_dtw_dyn.cuh (pairs pulled dynamically from a ring of staged utterances) == the static kernel == the reference's
    dtw, scores and first-wins argmin, over bank widths around the 32-template tile, all frame counts, mixed save_sign,
    the 2:1 guard, garbage headers; run twice so the second launch sees a dirty ring"""
    h = sr_b200.Handle(0)
    fin = sr_b200.synth_ftr_host(B, 0xD100 + T, fr[0], fr[1]).view(sr_b200.FTR_DTYPE).reshape(-1).copy()
    bank = sr_b200.synth_ftr_host(T, 0xD200 + T, fr[0], fr[1], stride=4096)
    rng = np.random.default_rng(T)
    bad = rng.random(T) < 0.2
    bank[bad, 0:2] = 0xFF
    if T > 3:
        bank[2, 2:4] = (200, 0)                            # frm_num 200 > vv_frm_max: never walked
        fin["frm_num"][1] = 0
        fin["frm_num"][2] = 300
    h.set_bank(bank, T, 4096)
    res = {}
    for v in (0, 1, 1):
        h.set_dtw_variant(v)
        res[v] = h.dtw(fin, flags=sr_b200.DTW_CHECK_SIGN)
        assert all(np.array_equal(a, b) for a, b in zip(res[v], res[0])), v
    ok = fin["frm_num"] <= 119
    want, _ = ora.dtw_batch(fin[ok], bank, T, 4096, check_sign=1)
    valid = np.ones(T, bool)
    if T > 3:
        valid[2] = False                                   # the reference would read past the struct: not comparable
    assert np.array_equal(res[1][0][ok][:, valid], want[:, valid])
    # through the recognise path (status gate: failed utterances never reach dtw)
    U = 8000
    pcm = sr_b200.synth_pcm_host(128, U, 0x77)
    pcm[::7] = 2048
    tb, _ = h.enrol(sr_b200.synth_pcm_host(min(T, 24), U, 0x7E3A0000), 2400)
    h.set_bank(tb, tb.shape[0], 4096)
    h.set_dtw_variant(0)
    a = h.recognise(pcm, 2400)
    h.set_dtw_variant(1)
    b = h.recognise(pcm, 2400)
    for k in ("score", "best_idx", "best_dis", "cmd", "status"):
        if k == "score":
            okr = a["status"] == 0
            assert np.array_equal(a[k][okr], b[k][okr])
        else:
            assert np.array_equal(a[k], b[k]), k
    h.close()


def test_dtw_extreme_values_wrap(handle, ora):
    """|dif| up to 65535 per dimension: the u32 accumulation of get_dis wraps (DTW.C:56)"""
    rng = np.random.default_rng(2)
    B, T = 40, 33
    ftr = sr_b200.synth_ftr_host(B, 1, 30, 60).view(sr_b200.FTR_DTYPE).reshape(-1).copy()
    ftr["mfcc_dat"] = rng.integers(-32768, 32768, ftr["mfcc_dat"].shape)
    bank = sr_b200.synth_ftr_host(T, 2, 30, 60)
    bank[:, 4:] = rng.integers(0, 256, bank[:, 4:].shape)
    handle.set_bank(bank, T, 2860)
    want, _ = ora.dtw_batch(ftr, bank, T, 2860)
    score, _, _ = handle.dtw(ftr)
    assert np.array_equal(score, want)
    a = rng.integers(-32768, 32768, (500, 12)).astype(np.int16)
    b = rng.integers(-32768, 32768, (500, 12)).astype(np.int16)
    assert np.array_equal(handle.get_dis(a, b), ora.get_dis(a, b))


@pytest.mark.parametrize("r", [10, 3, 15])
def test_dtw_band_extension_vs_own_dp_oracle(handle, r):
    """Sakoe-Chiba DP (BASELINE configs[2]); NOT in the reference -> checked against our own CPU DP (parity unpinned)"""
    B, T = 70, 45
    ftr = sr_b200.synth_ftr_host(B, 0xD7A00000, 1, 119).view(sr_b200.FTR_DTYPE).reshape(-1)
    ftr2 = sr_b200.synth_ftr_host(B, 0xD7A00100, 50, 100).view(sr_b200.FTR_DTYPE).reshape(-1)
    ftr = np.concatenate([ftr, ftr2])
    bank = sr_b200.synth_ftr_host(T, 0xD7A10000, 40, 110, stride=4096)
    handle.set_bank(bank, T, 4096)
    want, cells = ob.port().dtw_batch(ftr, bank, T, 4096, band_r=r, nthreads=4)
    score, bi, bd = handle.dtw(ftr, flags=sr_b200.DTW_BAND, band_r=r)
    assert np.array_equal(score, want) and cells > 0
    assert (want != ob.NULL).any() and (want == ob.NULL).any()
    key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
    assert np.array_equal(bd, (key.min(axis=1) >> np.uint64(32)).astype(np.uint32))
    # headers the banded kernels decode: unsigned and erased slots under the save_sign check, frm_num == 0 on both sides,
    # and one template with frm_num > vv_frm_max (never walked; the oracle would read past the struct, so its column is
    # checked directly and left out of the comparison)
    fin = ftr.copy()
    fin["frm_num"][:2] = 0
    bank2 = bank.copy()
    erased = np.random.default_rng(r).random(T) < 0.2
    erased[[3, 5]] = False
    bank2[erased, 0:2] = 0xFF
    bank2[1, 0:2] = 0                                      # unsigned
    bank2[3, 2:4] = 0                                      # frm_num 0
    bank2[5, 2:4] = (200, 0)                               # frm_num 200 > vv_frm_max
    handle.set_bank(bank2, T, 4096)
    score, bi, bd = handle.dtw(fin, flags=sr_b200.DTW_BAND | sr_b200.DTW_CHECK_SIGN, band_r=r)
    bank_o = bank2.copy()
    bank_o[5, 0:2] = 0xFF                                  # the oracle skips it under the save_sign check
    want, _ = ob.port().dtw_batch(fin, bank_o, T, 4096, check_sign=1, band_r=r, nthreads=4)
    cols = np.arange(T) != 5
    assert np.array_equal(score[:, cols], want[:, cols])
    assert (score[:, 5] == ob.NULL).all() and (score[:, erased | (np.arange(T) == 1)] == ob.NULL).all()
    assert (score[:2, 3] == ob.NULL).all() and (score[2:][:, cols] != ob.NULL).any()
    want[:, 5] = ob.NULL
    key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
    k = key.min(axis=1)
    assert np.array_equal(bi, (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)) and np.array_equal(bd, (k >> np.uint64(32)).astype(np.uint32))


# ---- spch_recg ---------------------------------------------------------------------------------------
def test_recognise_matches_golden_synthetic(handle):
    pcm = sr_b200.synth_pcm_host(24, 8000, 0x5EED0000)
    bank = GOLD["synth/bank"]
    handle.set_bank(bank, 8, 4096)
    out = handle.recognise(pcm, 2400)
    _cmp_recog(out, {k: GOLD["synth/" + k] for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status", "ftr")})
    pcm5 = sr_b200.synth_pcm_host(4, 40000, 0x5EED5000, 3)
    out5 = handle.recognise(pcm5, 2400)
    _cmp_recog(out5, {k: GOLD["synth5/" + k] for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status", "ftr")})


def test_recognise_mixed_failures_vs_oracle(handle, ora):
    rng = np.random.default_rng(6)
    B, U, T = 200, 8000, 11
    pcm = sr_b200.synth_pcm_host(B, U, 0xC0FFEE00)
    pcm[3] = 2048                                     # VAD fail
    pcm[4, 2500:7990] = rng.integers(0, 4096, 5490)   # segment never closes: VAD fail
    pcm[7] = rng.integers(0, 4096, U)
    tpl = sr_b200.synth_pcm_host(T, U, 0x7E3A0000)
    handle.set_bank(np.zeros((1, 4096), np.uint8), 0, 4096)
    e = handle.recognise(tpl, 2400, want=("ftr", "status"))
    bank = sr_b200.make_bank(e["ftr"], valid=[1, 1, 1, 0, 1, 1, 1, 1, 0, 1, 1])
    handle.set_bank(bank, T, 4096)
    out = handle.recognise(pcm, 2400)
    ref = ora.recognise_batch(pcm, 2400, bank, T, 4096)
    _cmp_recog(out, ref)
    assert set(out["status"].tolist()) >= {0, 1}
    # empty bank: idx 0, dis_max (main.c:276-278)
    handle.set_bank(bank, 0, 4096)
    o2 = handle.recognise(pcm[:5], 2400, want=("best_idx", "best_dis", "cmd"))
    assert (o2["best_idx"] == 0).all() and (o2["best_dis"] == ob.NULL).all()


def test_recognise_2s_buffers_and_long_segments(handle, ora):
    """the reference's native 2 s buffer; words long enough to exceed vv_frm_max -> MFCC fail (status 2)"""
    B, U = 16, 16000
    pcm = sr_b200.synth_pcm_host(B, U, 0x2222, 2)
    rng = np.random.default_rng(8)
    pcm[0, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    tpl = sr_b200.synth_pcm_host(4, 8000, 0x7E3A0000)
    handle.set_bank(np.zeros((1, 4096), np.uint8), 0, 4096)
    bank = sr_b200.make_bank(handle.recognise(tpl, 2400, want=("ftr",))["ftr"])
    handle.set_bank(bank, 4, 4096)
    out = handle.recognise(pcm, 2400)
    _cmp_recog(out, ora.recognise_batch(pcm, 2400, bank, 4, 4096))
    assert out["status"][0] == 2


# ---- the reference's own entry points (batch of 1) -----------------------------------------------------
def test_reference_named_entry_points(handle, ora):
    L = sr_b200.lib()
    pcm = CAPS["stm32_123"].copy()
    atap = np.zeros(1, sr_b200.ATAP_DTYPE)
    L.noise_atap(pcm.ctypes.data_as(C.c_void_p), 2400, atap.ctypes.data_as(C.c_void_p))
    assert atap.tobytes() == GOLD["stm32_123/atap"].tobytes()
    vv = (sr_b200.ValidTag * 3)()
    L.VAD(pcm.ctypes.data_as(C.c_void_p), 16000, vv, atap.ctypes.data_as(C.c_void_p))
    base = pcm.ctypes.data
    offs = [((v.start - base) // 2 if v.start else ob.NULL, (v.end - base) // 2 if v.end else ob.NULL) for v in vv]
    assert [x for p in offs for x in p] == GOLD["stm32_123/seg"].tolist()
    f = np.zeros(2, sr_b200.FTR_DTYPE)
    f["save_sign"] = 4321
    L.get_mfcc(C.byref(vv[0]), f[0:1].ctypes.data_as(C.c_void_p), atap.ctypes.data_as(C.c_void_p))
    L.get_mfcc(C.byref(vv[1]), f[1:2].ctypes.data_as(C.c_void_p), atap.ctypes.data_as(C.c_void_p))
    assert ob.ftr_equal(f[0:1], GOLD["stm32_123/ftr0"]) and ob.ftr_equal(f[1:2], GOLD["stm32_123/ftr1"])
    assert (f["save_sign"] == 4321).all()              # MFCC.C never writes save_sign
    d01 = L.dtw(f[0:1].ctypes.data_as(C.c_void_p), f[1:2].ctypes.data_as(C.c_void_p))
    d00 = L.dtw(f[0:1].ctypes.data_as(C.c_void_p), f[0:1].ctypes.data_as(C.c_void_p))
    assert [[d00, d01]] == GOLD["stm32_123/dtw"][:1].tolist()
    r0, r1 = f["mfcc_dat"][0][:12].copy(), f["mfcc_dat"][1][:12].copy()
    assert L.get_dis(r0.ctypes.data_as(C.c_void_p), r1.ctypes.data_as(C.c_void_p)) == ora.get_dis(r0.reshape(1, 12), r1.reshape(1, 12))[0]
    fr = (pcm[4000:4160].astype(np.int32) - 2213).astype(np.int16)
    p = L.fft(fr.ctypes.data_as(C.c_void_p), 160)
    mag = np.ctypeslib.as_array(p, shape=(1024,))[:512].copy()
    assert np.array_equal(mag, ora.fft_mag(fr.reshape(1, -1))[0])
    assert not L.fft(fr.ctypes.data_as(C.c_void_p), 1025)  # MFCC.C:32-35


# ---- full-size, size-independent properties ------------------------------------------------------------
def test_large_batch_shard_invariance_and_sampled_parity(handle, ora):
    """BASELINE-size run (16 384 x 1 s here to bound host RAM/time): results do not depend on how the batch is
    sharded (what the multi-GPU split relies on), enrolment then recognition of the same audio gives
    distance 0 against its own template, and a random sample agrees with the oracle bit-for-bit. Utterances whose
    segment starts at sample 0 sit on both sides of the chunk boundaries and of the cut."""
    B, U, T = 16384, 8000, 20
    pcm = sr_b200.synth_pcm_host(B, U, 0x5EED0000)
    planted = [2095, 2096, 4191, 4192, 4999, 5000]      # the host call's 32 MB chunks are 2 096 utterances; cut below
    ob.plant_sample0(pcm, planted, 0x5EED)
    handle.set_bank(np.zeros((1, 4096), np.uint8), 0, 4096)
    enrol = handle.recognise(pcm[:T], 2400, want=("ftr", "status"))
    assert (enrol["status"] == 0).all()
    bank = sr_b200.make_bank(enrol["ftr"])
    handle.set_bank(bank, T, 4096)
    full = handle.recognise(pcm, 2400)
    assert (full["best_idx"][:T] == np.arange(T)).all() and (full["best_dis"][:T] == 0).all()
    cut = 5000
    a = handle.recognise(pcm[:cut], 2400)
    b = handle.recognise(pcm[cut:], 2400)
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
        assert np.array_equal(full[k], np.concatenate([a[k], b[k]])), k
    assert ob.ftr_equal(full["ftr"], np.concatenate([a["ftr"], b["ftr"]]))
    idx = np.union1d(np.random.default_rng(0).choice(B, 192, replace=False), planted)
    ref = ob.recognise_pinned(ora, np.ascontiguousarray(pcm[idx]), 2400, bank, T, 4096)
    assert (ref["seg_off"][np.isin(idx, planted), 0, 0] == 0).all()
    _cmp_recog({k: v[idx] for k, v in full.items()}, ref)
    assert (full["status"] == 0).mean() > 0.99


# ---- x[-1] of a segment at sample 0: one rule for every batched path --------------------------------------
# VAD opens a segment at sample 0 when someone already speaks as the capture starts; get_mfcc then reads x[-1]
# (MFCC.C:119). Every batched entry point pins it to the utterance's own mid_val, so no result may depend on where
# the utterance sits: its row, the host call's chunks, a slice, the handles a batch is sharded over, another stream.
# Inputs: ob.plant_sample0 (reach and sensitivity are asserted in test_oracle.py); reference: ob.recognise_pinned.
def _sample0_bank(ora, T, geom_b=False):
    """T templates in flash layout, three of them short utterances whose segment starts at sample 0 (so planted
    utterances of 8..18 frames pass the 2:1 guard of DTW.C:133 against some templates)"""
    tpl = sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000)
    ob.plant_sample0(tpl, [1, 4, 7], 0x7E3A)
    e = ob.recognise_pinned(ob.port() if geom_b else ora, tpl, 2400, None, 0, 4096, geom_b=geom_b)
    assert (e["status"] == 0).all()
    return sr_b200.make_bank(e["ftr"])


def _same_recog(got, want, rows=None, what=""):
    """every field both dicts hold, bit for bit (features: the frm_num rows get_mfcc defines); `rows` selects the
    rows of `want` that `got` holds"""
    keys = [k for k in sr_b200.RECOG_FIELDS if k in got and k in want]
    assert {"seg_off", "ftr", "score", "best_idx", "best_dis", "cmd", "status"} <= set(keys), keys
    for k in keys:
        g, w = got[k], (want[k] if rows is None else want[k][rows])
        assert g.shape == w.shape, (what, k, g.shape, w.shape)
        if k == "ftr":
            bad = [i for i in range(len(g)) if not ob.ftr_equal(g[i:i + 1], w[i:i + 1])]
        elif k == "atap":
            bad = _first_bad_rows(g.view(np.uint8).reshape(len(g), -1), w.view(np.uint8).reshape(len(w), -1))
        else:
            bad = _first_bad_rows(g, w)
        assert not bad, (what, k, bad[:8])


def _planted_and_pinned(ora, pcm, rows, seed, bank, T):
    ob.plant_sample0(pcm, rows, seed)
    want = ob.recognise_pinned(ora, pcm, 2400, bank, T, 4096)
    planted = np.isin(np.arange(pcm.shape[0]), rows)
    assert ((want["seg_off"][:, 0, 0] == 0) == planted).all() and (want["status"][rows] == 0).all()
    return want


def test_mfcc_sample0_host_chunks_plain_packed_and_one_device_launch_agree(ora):
    """sr_recognise_batch runs a 32 MB chunk per launch: 256 utterances at U = 65 535, so 600 utterances are three
    chunks. Start-0 utterances at the first and last row of every chunk and a few others: the plain and the packed
    transport and one sr_recognise_batch_dev launch over the whole batch all equal recognise_pinned, every field"""
    B, U, T = 600, 65535, 9
    rng = np.random.default_rng(0x5A1)
    rows = sorted({0, 1, 2, 255, 256, 257, 511, 512, 513, 598, 599} | set(rng.choice(np.arange(3, 598), 5, replace=False).tolist()))
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A100000)
    bank = _sample0_bank(ora, T)
    want = _planted_and_pinned(ora, pcm, rows, 0x5A1, bank, T)
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    try:
        h.set_transport(0)
        plain = h.recognise(pcm, 2400)
        assert h.transport_stats()[:2] == (0, 3)
        h.set_transport(1)
        packed = h.recognise(pcm, 2400)
        assert sum(h.transport_stats()[:2]) == 3
    finally:
        h.set_transport(-1)
    hd = sr_b200.Handle(0)
    hd.set_bank(bank, T, 4096)
    one = recognise_dev_np(hd, pcm, 2400, T)
    _same_recog(plain, one, what="plain vs one launch")
    _same_recog(packed, plain, what="packed vs plain")
    _same_recog(one, want, what="one launch vs recognise_pinned")
    assert (want["best_dis"][rows] != ob.NULL).any()
    h.close()
    hd.close()


def test_mfcc_sample0_slices_and_single_utterances_equal_the_full_batch(handle, ora):
    """recognise(pcm[i:j]) with cuts at and next to start-0 utterances, and each of them as a batch of 1, equal the
    rows of the full batch, which equals recognise_pinned"""
    B, U, T = 64, 8000, 9
    rows = [0, 1, 2, 7, 8, 31, 32, 33, 62, 63]
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A200000)
    bank = _sample0_bank(ora, T)
    want = _planted_and_pinned(ora, pcm, rows, 0x5A2, bank, T)
    handle.set_bank(bank, T, 4096)
    full = handle.recognise(pcm, 2400)
    for i, j in ((1, 64), (2, 40), (7, 33), (8, 32), (9, 31), (31, 63), (32, 64), (33, 60)):
        _same_recog(handle.recognise(pcm[i:j], 2400), full, rows=slice(i, j), what=(i, j))
    for r in rows:
        _same_recog(handle.recognise(pcm[r:r + 1], 2400), full, rows=slice(r, r + 1), what=r)
    _same_recog(full, want, what="full vs recognise_pinned")


def test_mfcc_sample0_multi_handle_shards_equal_one_handle(ora):
    """sr_recognise_batch_multi over 2 and 3 handles (one GPU each when there are enough, else on GPU 0): shards start
    at B*g/n = 200, 300, 400, each of which, and the rows around it, holds a start-0 utterance"""
    import torch
    ng = max(1, torch.cuda.device_count())
    B, U, T = 600, 8000, 9
    rows = [0, 1, 199, 200, 201, 299, 300, 301, 399, 400, 401, 598, 599]
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A300000)
    bank = _sample0_bank(ora, T)
    want = _planted_and_pinned(ora, pcm, rows, 0x5A3, bank, T)
    h0 = sr_b200.Handle(0)
    h0.set_bank(bank, T, 4096)
    single = h0.recognise(pcm, 2400)
    for n in (2, 3):
        hs = [sr_b200.Handle(g % ng) for g in range(n)]
        for h in hs:
            h.set_bank(bank, T, 4096)
        multi = sr_b200.recognise_multi(hs, pcm, 2400, want=sr_b200.RECOG_FIELDS)
        _same_recog(multi, single, what=n)
        for h in hs:
            h.close()
    _same_recog(single, want, what="single vs recognise_pinned")
    h0.close()


def test_mfcc_sample0_enrol_whole_batch_equals_one_at_a_time(handle, ora):
    """sr_enrol_batch (pack_slots_kernel writes the flash slots): the whole batch gives the same slots and status as one
    utterance at a time, and the slots of recognise_pinned's features"""
    B, U = 40, 8000
    rows = [0, 1, 2, 5, 6, 20, 38, 39]
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A400000)
    pcm[10] = 2048                                     # VAD fails: the slot stays erased
    want = _planted_and_pinned(ora, pcm, rows, 0x5A4, None, 0)
    bank, status = handle.enrol(pcm, 2400)
    for b in range(B):
        one, st1 = handle.enrol(pcm[b:b + 1], 2400)
        assert np.array_equal(one[0], bank[b]) and st1[0] == status[b], b
    slots = sr_b200.make_bank(want["ftr"])
    slots[want["status"] != 0] = 0xFF
    assert np.array_equal(status, want["status"]) and status[10] == 1
    assert not _first_bad_rows(bank, slots), _first_bad_rows(bank, slots)


def _push_in_two_phases(pool, pcm, first, chunk=1000):
    """streams in `first` receive all their samples (chunks of `chunk`) while the others receive none; then the others"""
    S, L = pcm.shape
    events = []
    for group in (np.isin(np.arange(S), first), ~np.isin(np.arange(S), first)):
        for n0 in range(0, L, chunk):
            w = min(chunk, L - n0)
            lens = np.where(group, w, 0).astype(np.uint32)
            events += pool.push_ragged(np.ascontiguousarray(pcm[:, n0:n0 + w]), lens)
    return events


def _check_sample0_events(events, want, batch, planted):
    """events == the closed segments of recognise_pinned's VAD; segment 0's results == recognise_pinned == the batch"""
    S = want["status"].shape[0]
    closed = [(s, k) for s in range(S) for k in range(3) if want["seg_off"][s, k, 1] != ob.NULL]
    assert sorted((e["stream"], e["segment"]) for e in events) == closed
    seen = set()
    for e in events:
        s, k = e["stream"], e["segment"]
        assert (e["start"], e["end"]) == tuple(want["seg_off"][s, k])
        if k == 0:
            seen.add(s)
            got = (e["frm_num"], e["status"], e["best_idx"], e["best_dis"], e["cmd"])
            b = tuple(int(batch[q][s]) for q in ("status", "best_idx", "best_dis", "cmd"))
            assert got[1:] == b, ("event vs batch", e, b)
            w = (int(want["ftr"]["frm_num"][s]), int(want["status"][s]), int(want["best_idx"][s]), int(want["best_dis"][s]), int(want["cmd"][s]))
            assert got == w, ("event vs recognise_pinned", e, w)
    assert set(planted) <= seen


@pytest.mark.parametrize("group", [False, True], ids=["one_handle", "group_of_two"])
def test_mfcc_sample0_streaming_events_equal_pinned_and_batch(ora, group):
    """one stream per utterance, start-0 utterances in streams s >= 1 (row s of the pool's [S][L] buffer, after stream
    s-1's row). First the row before is still unfilled when the segment closes (stream s-1 is pushed after s), then,
    after reset() and with other contents, it is already full. Events equal recognise_pinned and the batch call; with
    a stream group of two handles the streams are sharded over both"""
    S, L, T = 8, 8000, 9
    bank = _sample0_bank(ora, T)
    hs = [sr_b200.Handle(0) for _ in range(2 if group else 1)]
    for h in hs:
        h.set_bank(bank, T, 4096)
    pool = sr_b200.StreamPool(hs if group else hs[0], S, L, 2400)
    for run, (planted, first) in enumerate((([1, 3, 5, 7], [1, 3, 5, 7]),          # stream s-1 empty when s closes
                                            ([2, 4, 6], [0, 1, 3, 5, 7]))):       # stream s-1 already full
        if run:
            pool.reset()
        pcm = sr_b200.synth_pcm_host(S, L, 0x5A500000 + 0x100 * run)
        want = _planted_and_pinned(ora, pcm, planted, 0x5A5 + run, bank, T)
        batch = hs[0].recognise(pcm, 2400)
        events = _push_in_two_phases(pool, pcm, first)
        _check_sample0_events(events, want, batch, planted)
        _same_recog(batch, want, what=run)
        seg, atap = pool.segments()
        assert np.array_equal(seg, want["seg_off"]) and atap.tobytes() == want["atap"].tobytes()
    pool.close()
    for h in hs:
        h.close()


def test_geom_b_sample0_batch_and_streaming_pin_mid_val():
    """GEOM_B (mfcc_geomb_kernel) follows the same rule: get_mfcc of start-0 segments in every row, the recognise path
    and streaming equal the port's GEOM_B restatement on [mid_val, row...] rows (parity unpinned, as for every GEOM_B
    test)"""
    po = ob.port()
    h = sr_b200.Handle(0)
    h.set_geometry(1)
    B, U, T = 24, 8000, 9
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A600000)
    pcm[:, -1] = np.where(np.arange(B) % 2 == 0, 0, 4095)
    seg = np.tile(np.array([0, 1600], np.uint32), (B, 1))
    seg[3] = (1, 1601)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2048
    atap["mid_val"][5] = 300
    want_f = po.mfcc_geom_b_batch(ob.pinned_rows(pcm, atap), seg + 1, atap)
    assert (want_f["frm_num"] == 18).all()
    assert ob.ftr_equal(h.mfcc(pcm, seg, atap), want_f)
    bank = _sample0_bank(None, T, geom_b=True)
    h.set_bank(bank, T, 4096)
    rows = [0, 1, 2, 5, 11, 12, 17, 22, 23]
    ob.plant_sample0(pcm, rows, 0x5A6)
    want = ob.recognise_pinned(po, pcm, 2400, bank, T, 4096, geom_b=True)
    assert (want["seg_off"][rows, 0, 0] == 0).all() and (want["status"][rows] == 0).all()
    batch = h.recognise(pcm, 2400)
    pool = sr_b200.StreamPool(h, B, U, 2400)
    events = _push_in_two_phases(pool, pcm, rows)
    pool.close()
    _check_sample0_events(events, want, batch, rows)
    _same_recog(batch, want, what="batch")
    h.close()


# ---- device-pointer variants on a torch stream ----------------------------------------------------------
def test_device_pointer_api_on_torch_stream(ora):
    import torch
    dev = torch.device("cuda:0")
    B, U, T = 300, 8000, 9
    h = sr_b200.Handle(0)
    st = torch.cuda.Stream(dev)
    h.set_stream(st.cuda_stream)
    pcm_h = sr_b200.synth_pcm_host(B, U, 0x5151)
    with torch.cuda.stream(st):
        pcm = torch.empty((B, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(pcm.data_ptr(), B, U, 0x5151, 1, st.cuda_stream)     # device generator == host generator
        tpl = torch.empty((T, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(tpl.data_ptr(), T, U, 0x7E3A0000, 1, st.cuda_stream)
        ftr_t = torch.zeros((T, 2860), dtype=torch.uint8, device=dev)
        h.set_bank_dev(0, 0, 4096)
        h.recognise_dev(tpl.data_ptr(), U, T, 2400, ftr=ftr_t.data_ptr())
        bank = torch.full((T, 4096), 255, dtype=torch.uint8, device=dev)
        bank[:, :2860] = ftr_t
        bank[:, 0] = 12345 & 0xFF
        bank[:, 1] = 12345 >> 8
        h.set_bank_dev(bank.data_ptr(), T, 4096)
        score = torch.zeros((B, T), dtype=torch.int32, device=dev)
        bidx = torch.zeros(B, dtype=torch.int32, device=dev)
        bdis = torch.zeros(B, dtype=torch.int32, device=dev)
        cmd = torch.zeros(B, dtype=torch.int32, device=dev)
        status = torch.zeros(B, dtype=torch.uint8, device=dev)
        seg = torch.zeros((B, 6), dtype=torch.int32, device=dev)
        h.recognise_dev(pcm.data_ptr(), U, B, 2400, seg_off=seg.data_ptr(), score=score.data_ptr(),
                        best_idx=bidx.data_ptr(), best_dis=bdis.data_ptr(), cmd=cmd.data_ptr(), status=status.data_ptr())
    st.synchronize()
    assert np.array_equal(pcm.cpu().numpy().view(np.uint16), pcm_h)
    bank_h = bank.cpu().numpy()
    ref = ora.recognise_batch(pcm_h, 2400, bank_h, T, 4096)
    assert np.array_equal(score.cpu().numpy().view(np.uint32), ref["score"])
    assert np.array_equal(seg.cpu().numpy().view(np.uint32).reshape(-1), ref["seg_off"].reshape(-1))
    assert np.array_equal(bidx.cpu().numpy().view(np.uint32), ref["best_idx"])
    assert np.array_equal(bdis.cpu().numpy().view(np.uint32), ref["best_dis"])
    assert np.array_equal(cmd.cpu().numpy().view(np.uint32), ref["cmd"])
    assert np.array_equal(status.cpu().numpy(), ref["status"])
    assert h.launch_count() >= 6
    h.close()


def _to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to("cuda:0")


@pytest.mark.parametrize("U", [8000, 8003, 16000])
def test_unaligned_device_pcm_vad_mfcc_recognise(ora, U):
    """the _dev entry points take pcm with 2-byte alignment (speech_recog.h). A batch base that is not 16-byte aligned makes
    vad_kernel stage with plain loads (chunk_issue) and mfcc_kernel with its cooperative copy (stage_utterance), which
    must pin x[-1] of a segment at sample 0 to mid_val as the bulk copy does; noise windows past 2 560 samples read global
    memory from the unaligned base"""
    import torch
    dev = torch.device("cuda:0")
    B, T = 40, 8
    pcm = sr_b200.synth_pcm_host(B, U, 0xA1160000 + U, 1 if U < 16000 else 2)
    rng = np.random.default_rng(U)
    pcm[3] = 2048                                      # VAD fails
    pcm[5] = rng.integers(0, 65536, U)                 # full range
    # MFCC segments: ragged, 1 frame, < 1 frame, 119 and 120 frames where U allows, NULL, ending at the batch end
    st_ = rng.integers(1, 900, B)
    seg = np.stack([st_, np.minimum(st_ + rng.integers(160, 4000, B), U)], 1).astype(np.uint32)
    seg[0] = (0, 1600)                                 # x[-1] of the whole batch: pinned to mid_val
    seg[1] = (1, 161)
    seg[2] = (7, 7 + 159)
    seg[4] = (ob.NULL, ob.NULL)
    if U >= 2 + 119 * 80 + 160:
        seg[6] = (1, 1 + 118 * 80 + 160)
        seg[7] = (2, 2 + 119 * 80 + 160)
    seg[B - 1] = (U - 1999, U)
    atm = np.zeros(B, sr_b200.ATAP_DTYPE)
    atm["mid_val"] = rng.integers(0, 4096, B)
    atm["mid_val"][0] = 2100
    valid = (seg != ob.NULL).all(axis=1)
    # oracle rows of U + 1 samples: row b's own samples after the sample before them in the contiguous batch (mid_val for
    # row 0), i.e. x[-1] as the kernel sees it
    flat = np.concatenate([[np.uint16(2100)], pcm.reshape(-1)])
    rows1 = np.stack([flat[b * U: b * U + U + 1] for b in range(B)])
    want_f = ora.mfcc_batch(rows1[valid], seg[valid] + 1, atm[valid])
    fv = want_f["frm_num"]
    assert fv[0] == 19 and fv[1] == 1 and fv[2] == 0 and (U < 2 + 119 * 80 + 160 or (fv[5] == 119 and fv[6] == 0))
    want_a = {n_len: np.concatenate([ora.noise_atap(pcm[b], n_len) for b in range(B)]) for n_len in (2400, 4800)}
    want_s = np.stack([ora.vad(pcm[b], U, want_a[2400][b:b + 1]) for b in range(B)])
    tpl = sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000)
    h = sr_b200.Handle(0)
    bank, est = h.enrol(tpl, 2400)
    assert (est == 0).all()
    h.set_bank(bank, T, 4096)
    want_r = ora.recognise_batch(pcm, 2400, bank, T, 4096)
    assert set(want_r["status"].tolist()) >= {0, 1}
    st = torch.cuda.Stream(dev)
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        buf = torch.zeros(B * U + 16, dtype=torch.int16, device=dev)
        seg_d, atm_d = _to_dev(seg), _to_dev(atm)
        for k in (1, 3, 7):
            buf.zero_()
            buf[k:k + B * U] = torch.from_numpy(pcm.view(np.int16).reshape(-1)).to(dev)
            ptr = buf.data_ptr() + 2 * k
            assert ptr % 16 != 0
            for n_len in (2400, 4800):
                at = torch.full((B * 12,), 0xA5, dtype=torch.uint8, device=dev)
                h.noise_atap_dev(ptr, U, B, n_len, at.data_ptr())
                st.synchronize()
                assert at.cpu().numpy().tobytes() == want_a[n_len].tobytes(), (k, n_len)
            sg = torch.full((B * 6,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
            h.vad_dev(ptr, U, B, U, at.data_ptr(), sg.data_ptr())        # atap of the 4 800-sample window
            st.synchronize()
            want_s48 = np.stack([ora.vad(pcm[b], U, want_a[4800][b:b + 1]) for b in range(B)])
            assert np.array_equal(sg.cpu().numpy().view(np.uint32).reshape(B, 6), want_s48), k
            ft = torch.full((B * sr_b200.FTR_BYTES,), 0x5A, dtype=torch.uint8, device=dev)
            h.mfcc_dev(ptr, U, B, seg_d.data_ptr(), 2, atm_d.data_ptr(), ft.data_ptr())
            st.synchronize()
            got_f = ft.cpu().numpy().view(sr_b200.FTR_DTYPE)
            assert ob.ftr_equal(got_f[valid], want_f) and (got_f["frm_num"][~valid] == 0).all(), k
            out = {"atap": torch.full((B * 12,), 0xA5, dtype=torch.uint8, device=dev),
                   "seg_off": torch.full((B * 6,), 0x5A5A5A5A, dtype=torch.int32, device=dev),
                   "ftr": torch.full((B * sr_b200.FTR_BYTES,), 0x5A, dtype=torch.uint8, device=dev),
                   "score": torch.full((B * T,), 0x5A5A5A5A, dtype=torch.int32, device=dev),
                   "status": torch.full((B,), 0x5A, dtype=torch.uint8, device=dev)}
            for key in ("best_idx", "best_dis", "cmd"):
                out[key] = torch.full((B,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
            h.recognise_dev(ptr, U, B, 2400, **{key: v.data_ptr() for key, v in out.items()})
            st.synchronize()
            got = {key: v.cpu().numpy() for key, v in out.items()}
            assert got["atap"].tobytes() == want_a[2400].tobytes(), k
            assert np.array_equal(got["seg_off"].view(np.uint32).reshape(B, 6), want_s), k
            got["ftr"] = got["ftr"].view(sr_b200.FTR_DTYPE)
            got["seg_off"] = got["seg_off"].view(np.uint32)
            for key in ("score", "best_idx", "best_dis", "cmd"):
                got[key] = got[key].view(np.uint32)
            _cmp_recog(got, want_r)
    h.close()


@pytest.mark.parametrize("stride", [4096, 2860])
def test_device_bank_wider_than_one_tile_rewritten_in_place(ora, stride):
    """sr_set_bank_dev with T = 70 > 32: the headers come back with a strided D2H copy and the slots are walked in
    ascending frm_num order. Rewriting the bank in place (slots permuted, frm_num changed, signs erased) and setting the same
    pointer again keeps the stale order, which may only cost speed: results equal the oracle on the new contents"""
    import torch
    dev = torch.device("cuda:0")
    B, U, T = 96, 8000, 70
    h = sr_b200.Handle(0)
    bank, est = h.enrol(sr_b200.synth_pcm_host(T, U, 0x7E3A0000 + stride), 2400, slot_stride=stride)
    assert (est == 0).all()
    rng = np.random.default_rng(stride)
    bad = rng.random(T) < 0.25
    bank[bad, 0:2] = 0xFF                              # erased flash: save_sign != 12345
    bank[np.nonzero(~bad)[0][:3], 0:2] = 0             # another wrong sign
    pcm = sr_b200.synth_pcm_host(B, U, 0xBA2C0000 + stride)
    pcm[::11] = 2048                                   # VAD fails
    fin = sr_b200.synth_ftr_host(B, 0xBA2D0000 + stride, 1, 119).view(sr_b200.FTR_DTYPE).reshape(-1)

    def order(b):                                      # the walk order sr_set_bank_dev derives from the headers
        f = b[:, 2].astype(np.int64) | (b[:, 3].astype(np.int64) << 8)
        return np.argsort(np.where(f > 119, 0xFFFF, f), kind="stable")

    def check(bank_h):
        out = {"score": torch.zeros((B, T), dtype=torch.int32, device=dev)}
        for key in ("best_idx", "best_dis", "cmd"):
            out[key] = torch.zeros(B, dtype=torch.int32, device=dev)
        out["status"] = torch.zeros(B, dtype=torch.uint8, device=dev)
        h.recognise_dev(pcm_d.data_ptr(), U, B, 2400, **{key: v.data_ptr() for key, v in out.items()})
        st.synchronize()
        ref = ora.recognise_batch(pcm, 2400, bank_h, T, stride)
        for key, v in out.items():
            assert np.array_equal(v.cpu().numpy().view(ref[key].dtype).reshape(ref[key].shape), ref[key]), key
        assert (ref["status"] == 0).sum() > B // 2 and (ref["score"][ref["status"] == 0] != ob.NULL).any()
        score, bi, bd = h.dtw(fin, flags=sr_b200.DTW_CHECK_SIGN)
        want, _ = ora.dtw_batch(fin, bank_h, T, stride, check_sign=1)
        assert np.array_equal(score, want)
        key64 = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
        kmin = key64.min(axis=1)
        assert np.array_equal(bi, (kmin & np.uint64(0xFFFFFFFF)).astype(np.uint32))
        assert np.array_equal(bd, (kmin >> np.uint64(32)).astype(np.uint32))

    st = torch.cuda.Stream(dev)
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        pcm_d = torch.from_numpy(pcm.view(np.int16)).to(dev)
        bank_d = _to_dev(bank)
        ptr = bank_d.data_ptr()
        assert T > 32
        h.set_bank_dev(ptr, T, stride)
        check(bank)
        # in place: permute the slots, shorten / lengthen some templates (rows past the old end are erased flash), erase signs
        new = bank[rng.permutation(T)].copy()
        for t in rng.choice(T, 12, replace=False):
            f = int(rng.integers(1, 120))
            new[t, 2], new[t, 3] = f & 0xFF, f >> 8
        new[rng.choice(T, 5, replace=False), 0:2] = 0xFF
        assert not np.array_equal(order(new), order(bank))
        bank_d.copy_(_to_dev(new))
        assert bank_d.data_ptr() == ptr
        h.set_bank_dev(ptr, T, stride)                 # the same buffer: the order of the old contents is kept
        check(new)
    h.close()


def test_enrol_and_get_mdl(handle, ora):
    """save_mdl (main.c:121-138 + Flash.C:17-67) as a batch, and the reference's template averaging get_mdl"""
    B, U = 40, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0x7E3A0000)
    pcm[5] = 2048                                     # VAD_fail: slot stays erased
    bank, status = handle.enrol(pcm, 2400)
    ref = ora.recognise_batch(pcm, 2400, None, 0, 4096)
    assert np.array_equal(status, ref["status"]) and status[5] == 1
    want = sr_b200.make_bank(ref["ftr"])
    want[ref["status"] != 0] = 0xFF                   # save_ftr_mdl is never reached: the slot stays erased
    assert np.array_equal(bank, want) and (bank[5] == 0xFF).all()
    f1 = sr_b200.synth_ftr_host(64, 0xAA00, 1, 59).view(sr_b200.FTR_DTYPE).reshape(-1)
    f2 = sr_b200.synth_ftr_host(64, 0xBB00, 1, 59).view(sr_b200.FTR_DTYPE).reshape(-1)
    want_m, want_d = ora.get_mdl(f1, f2)
    pre = np.zeros(64, sr_b200.FTR_DTYPE)
    pre["save_sign"] = 777
    got_m, got_d = handle.get_mdl(f1, f2, pre)
    assert np.array_equal(got_d, want_d) and ob.ftr_equal(got_m, want_m) and (got_m["save_sign"] == 777).all()
    # long paths: frm_num clamps at 119 instead of the reference's out-of-bounds writes (port == kernel)
    g1 = sr_b200.synth_ftr_host(16, 0xCC00, 100, 119).view(sr_b200.FTR_DTYPE).reshape(-1)
    g2 = sr_b200.synth_ftr_host(16, 0xDD00, 100, 119).view(sr_b200.FTR_DTYPE).reshape(-1)
    pm, pd = ob.port().get_mdl(g1, g2)
    gm, gd = handle.get_mdl(g1, g2)
    assert np.array_equal(gd, pd) and ob.ftr_equal(gm, pm) and (gm["frm_num"] == 119).any()


@pytest.mark.parametrize("chunk", [80, 800, 777])
def test_streaming_equals_batch(handle, ora, chunk):
    """lock-step chunked capture (config 5 shape: 5 s streams, 3 words): the union of the streaming events equals
    the batch VAD on the finished buffers, and every event equals get_mfcc + dtw of that segment"""
    S, L, T = 24, 40000, 8
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EED5000, 3)
    pcm[3] = 2048                                     # a silent stream: no event
    bank = GOLD["synth/bank"]
    handle.set_bank(bank, T, 4096)
    pool = sr_b200.StreamPool(handle, S, L, 2400)
    events, latest = [], {}
    pin_ptr = None
    if chunk == 800:                                   # pinned capture array: chunks are read zero-copy, strided ([S][L] rows)
        arr, pin_ptr = sr_b200.host_alloc_dev(0, S * L * 2)
        arr.view(np.uint16).reshape(S, L)[:] = pcm
    for n0 in range(0, L, chunk):
        c = np.ascontiguousarray(pcm[:, n0:n0 + chunk])
        evs = pool.push(pin_ptr + 2 * n0, c.shape[1], L) if pin_ptr else pool.push(c)
        for e in evs:
            # the segment closes with the chunk that delivers sample end+879 (last sample of the closing frame)
            assert n0 <= e["end"] + 879 < n0 + c.shape[1]
        events += evs
    seg, atap = pool.segments()
    pool.close()
    if pin_ptr:
        sr_b200.host_free(pin_ptr)
    batch_atap = handle.noise_atap(pcm, 2400)
    assert atap.tobytes() == batch_atap.tobytes()
    batch_seg = handle.vad(pcm, batch_atap)
    assert np.array_equal(seg, batch_seg)
    closed = [(s, k) for s in range(S) for k in range(3) if batch_seg[s, k, 1] != ob.NULL]
    assert sorted((e["stream"], e["segment"]) for e in events) == closed and len(closed) >= 3 * (S - 1) - 2
    for e in events:
        s, k = e["stream"], e["segment"]
        assert (e["start"], e["end"]) == tuple(batch_seg[s, k])
        f = ora.mfcc_batch(pcm[s:s + 1], batch_seg[s, k].reshape(1, 2), batch_atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]) and e["status"] == 0
        sc, _ = ora.dtw_batch(f, bank, T, 4096, check_sign=1)
        key = (sc[0].astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)
        assert e["best_dis"] == int(key.min() >> np.uint64(32)) and e["best_idx"] == int(key.min() & np.uint64(0xFFFFFFFF))
        assert e["cmd"] == e["best_idx"] // 4


def _check_stream_events(handle, ora, pcm, bank, T, events, seg, atap):
    S = pcm.shape[0]
    batch_atap = handle.noise_atap(pcm, 2400)
    assert atap.tobytes() == batch_atap.tobytes()
    batch_seg = handle.vad(pcm, batch_atap)
    assert np.array_equal(seg, batch_seg)
    closed = [(s, k) for s in range(S) for k in range(3) if batch_seg[s, k, 1] != ob.NULL]
    assert sorted((e["stream"], e["segment"]) for e in events) == closed and len(closed) >= 2 * S
    want = handle.recognise(pcm, 2400, want=("best_idx", "best_dis", "cmd", "status"))     # segment 0 == the batch call
    for e in events:
        s, k = e["stream"], e["segment"]
        assert (e["start"], e["end"]) == tuple(batch_seg[s, k])
        if k == 0:
            assert (e["best_idx"], e["best_dis"], e["cmd"], e["status"]) == tuple(int(want[q][s]) for q in ("best_idx", "best_dis", "cmd", "status"))
    for e in events[:: max(1, len(events) // 12)]:           # a sample against the oracle, segment by segment
        s, k = e["stream"], e["segment"]
        f = ora.mfcc_batch(pcm[s:s + 1], batch_seg[s, k].reshape(1, 2), batch_atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]) and e["status"] == 0
        sc, _ = ora.dtw_batch(f, bank, T, 4096, check_sign=1)
        key = (sc[0].astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)
        assert e["best_dis"] == int(key.min() >> np.uint64(32)) and e["best_idx"] == int(key.min() & np.uint64(0xFFFFFFFF))


def test_streaming_ragged_arrival_equals_batch(handle, ora):
    """every stream advances at its own pace (random chunk lengths incl. 0 and odd ones, some streams far ahead of
    others, a stream that starts late): events and final segments still equal the batch results"""
    S, L, T = 40, 40000, 8
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EED6000, 3)
    bank = GOLD["synth/bank"]
    handle.set_bank(bank, T, 4096)
    pool = sr_b200.StreamPool(handle, S, L, 2400)
    rng = np.random.default_rng(77)
    pos = np.zeros(S, np.int64)
    events, pushes = [], 0
    while (pos < L).any():
        lens = rng.choice([0, 1, 79, 80, 81, 160, 333, 800, 1601, 4000], S).astype(np.int64)
        lens[5] = 0 if pushes < 30 else lens[5]            # stream 5 starts late
        lens = np.minimum(lens, L - pos)
        w = int(lens.max())
        if w == 0:
            continue
        chunk = np.zeros((S, w), np.uint16)
        for s in range(S):
            chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
        evs = pool.push_ragged(chunk, lens)
        for e in evs:                                       # an event appears with the push that delivers sample end+879
            s = e["stream"]
            assert pos[s] <= e["end"] + 879 < pos[s] + lens[s], (e, pos[s], lens[s])
        events += evs
        pos += lens
        pushes += 1
    seg, atap = pool.segments()
    pool.close()
    _check_stream_events(handle, ora, pcm, bank, T, events, seg, atap)


def test_streaming_small_event_buffer_keeps_events(handle, ora):
    """max_events smaller than what a push closes: nothing is lost, the rest comes with later pushes / sr_streams_fetch"""
    S, L, T = 32, 16000, 8
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EED7000, 1)
    handle.set_bank(GOLD["synth/bank"], T, 4096)
    pool = sr_b200.StreamPool(handle, S, L, 2400)
    full = []
    for n0 in range(0, L, 4000):
        full += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 4000]))
    pool.reset()
    got = []
    for n0 in range(0, L, 4000):
        evs = pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 4000]), max_events=3)
        assert len(evs) <= 3
        got += evs
    assert pool.pending() == len(full) - len(got) > 0
    while pool.pending():
        got += pool.fetch(max_events=5)
    pool.close()
    key = lambda e: (e["stream"], e["segment"])             # the order inside one push is the order the warps finished
    assert sorted(got, key=key) == sorted(full, key=key) and len(full) >= S - 2


def test_stream_group_shards_streams_over_handles(handle, ora):
    """sr_stream_group: streams sharded over several handles (all visible GPUs, or two handles on one GPU), lock-step and
    ragged pushes; events carry global stream numbers and equal the batch results"""
    import torch
    ng = max(1, torch.cuda.device_count())
    devs = list(range(ng)) if ng > 1 else [0, 0]
    S, L, T = 37, 40000, 8
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EED8000, 3)
    bank = GOLD["synth/bank"]
    hs = [sr_b200.Handle(d) for d in devs]
    for h in hs:
        h.set_bank(bank, T, 4096)
    handle.set_bank(bank, T, 4096)
    pool = sr_b200.StreamPool(hs, S, L, 2400)
    events = []
    for n0 in range(0, 20000, 800):
        events += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 800]))
    rng = np.random.default_rng(5)
    pos = np.full(S, 20000, np.int64)
    while (pos < L).any():
        lens = np.minimum(rng.integers(0, 1500, S), L - pos)
        w = max(int(lens.max()), 1)
        chunk = np.zeros((S, w), np.uint16)
        for s in range(S):
            chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
        events += pool.push_ragged(chunk, lens)
        pos += lens
    seg, atap = pool.segments()
    pool.close()
    _check_stream_events(handle, ora, pcm, bank, T, events, seg, atap)
    for h in hs:
        h.close()


def test_geom_b_extension_vs_own_oracle():
    """GEOM_B (200/80/256, BASELINE configs[0]'s framing): PARITY UNPINNED -- the reference has no 256-point path, the
    checker is this repo's own restatement (oracle/sr_oracle.c::sro_mfcc_geom_b, whose FFT generalisation is pinned at
    N = 1024). get_mfcc alone on synthetic / full-range / ragged segments, then the whole recognise path"""
    po = ob.port()
    h = sr_b200.Handle(0)
    h.set_geometry(1)
    B, U = 96, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0xB0B0)
    rng = np.random.default_rng(0xB)
    pcm[80:] = rng.integers(0, 65536, (16, U)).astype(np.uint16)          # full-range samples: s16 / u32 wraps
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2048
    atap["mid_val"][80:] = rng.integers(0, 65536, 16)
    seg = np.zeros((B, 2), np.uint32)
    seg[:, 0] = 80 * rng.integers(1, 30, B)
    seg[:, 1] = np.minimum(seg[:, 0] + 80 * rng.integers(1, 100, B), U)
    seg[1] = (80, 80 + 199)                                                # shorter than one 200-sample frame
    seg[2] = (80, 280)                                                     # exactly one frame
    seg[3] = (80, 80 + 200 + 80 * 119)                                     # 120 frames: rejected (vv_frm_max)
    seg[4] = (0xFFFFFFFF, 0xFFFFFFFF)
    seg[5] = (160, 8000)
    got = h.mfcc(pcm, seg, atap)
    want = po.mfcc_geom_b_batch(pcm, seg, atap)
    assert ob.ftr_equal(got, want)
    assert int(got["frm_num"][2]) == 1 and int(got["frm_num"][1]) == 0 and int(got["frm_num"][3]) == 0 and int(got["frm_num"][5]) == 96
    assert (got["frm_num"] > 0).sum() > 60
    # the same frames in the reference geometry are different numbers (this is a different front end, not a re-labelling)
    h.set_geometry(0)
    ref_geom = h.mfcc(pcm, seg, atap)
    assert not ob.ftr_equal(ref_geom, got)
    # whole path: enrol + recognise in GEOM_B == VAD (reference framing) -> GEOM_B features -> dtw -> argmin on the CPU
    h.set_geometry(1)
    T = 6
    tpl = sr_b200.synth_pcm_host(T, U, 0x7E3A0000)
    bank, est = h.enrol(tpl, 2400)
    assert (est == 0).all()
    h.set_bank(bank, T, 4096)
    utt = sr_b200.synth_pcm_host(32, U, 0x5EED0000)
    out = h.recognise(utt, 2400)
    a = np.zeros(32, sr_b200.ATAP_DTYPE)
    for b in range(32):
        a[b] = po.noise_atap(utt[b], 2400)[0]
    sg = np.stack([po.vad(utt[b], U, a[b:b + 1]) for b in range(32)]).reshape(32, 3, 2)
    assert np.array_equal(out["seg_off"], sg)
    f = po.mfcc_geom_b_batch(utt, sg[:, 0, :], a)
    ok = sg[:, 0, 1] != ob.NULL
    assert ob.ftr_equal(out["ftr"][ok], f[ok])
    sc, _ = po.dtw_batch(f, bank, T, 4096, check_sign=1)
    assert np.array_equal(out["score"][ok], sc[ok]) and ok.sum() >= 30
    h.close()


@pytest.mark.parametrize("arrival", ["lockstep", "ragged"])
def test_geom_b_streaming_vs_own_oracle(ora, arrival):
    """streaming pushes on a handle in GEOM_B go to mfcc_geomb_kernel with a row map and a batch size produced on the
    device: every event equals the port's VAD, then GEOM_B get_mfcc, dtw and argmin of that segment (parity unpinned, as
    for the batch GEOM_B test)"""
    po = ob.port()
    h = sr_b200.Handle(0)
    h.set_geometry(1)
    S, L, T = 24, 40000, 6
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDB000, 3)
    pcm[3] = 2048                                      # a silent stream: no event
    bank, est = h.enrol(sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000), 2400)
    assert (est == 0).all()
    h.set_bank(bank, T, 4096)
    pool = sr_b200.StreamPool(h, S, L, 2400)
    events = []
    if arrival == "lockstep":
        for n0 in range(0, L, 800):
            events += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 800]))
    else:
        rng = np.random.default_rng(0xB5)
        pos = np.zeros(S, np.int64)
        while (pos < L).any():
            lens = np.minimum(rng.choice([0, 1, 79, 81, 160, 333, 1601, 4000], S), L - pos)
            w = int(lens.max())
            if w == 0:
                continue
            chunk = np.zeros((S, w), np.uint16)
            for s in range(S):
                chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
            events += pool.push_ragged(chunk, lens)
            pos += lens
    seg, atap = pool.segments()
    pool.close()
    for s in range(S):
        a = po.noise_atap(pcm[s], 2400)
        assert a.tobytes() == atap[s:s + 1].tobytes(), s
        assert po.vad(pcm[s], L, a).tolist() == seg[s].reshape(-1).tolist(), s
    closed = [(s, k) for s in range(S) for k in range(3) if seg[s, k, 1] != ob.NULL]
    assert sorted((e["stream"], e["segment"]) for e in events) == closed and len(closed) >= 2 * S
    geometry_differs = 0
    for e in events:
        s, k = e["stream"], e["segment"]
        assert (e["start"], e["end"]) == tuple(seg[s, k])
        f = po.mfcc_geom_b_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]), e
        if e["frm_num"] == 0:
            assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (2, 0, ob.NULL, 0), e
            continue
        sc, _ = po.dtw_batch(f, bank, T, 4096, check_sign=1)
        kmin = ((sc[0].astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)).min()
        assert e["status"] == 0 and e["best_dis"] == int(kmin >> np.uint64(32)), e
        assert e["best_idx"] == int(kmin & np.uint64(0xFFFFFFFF)) and e["cmd"] == e["best_idx"] // 4, e
        ref_geom = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
        geometry_differs += int(ref_geom["frm_num"][0]) != e["frm_num"]
    assert geometry_differs > 0                        # the 200-sample framing ran, not the reference's 160
    h.close()


def test_recognise_multi_handle_sharding(ora):
    """sr_recognise_batch_multi: contiguous shards over several handles (all visible GPUs, or two handles on one GPU)
    == the single-handle result, bit for bit"""
    import torch
    ng = max(1, torch.cuda.device_count())
    devs = list(range(ng)) if ng > 1 else [0, 0]
    B, U, T = 1003, 8000, 9
    pcm = sr_b200.synth_pcm_host(B, U, 0x3131)
    hs = [sr_b200.Handle(d) for d in devs]
    bank, _ = hs[0].enrol(sr_b200.synth_pcm_host(T, U, 0x7E3A0000), 2400)
    for h in hs:
        h.set_bank(bank, T, 4096)
    multi = sr_b200.recognise_multi(hs, pcm, 2400)
    single = hs[0].recognise(pcm, 2400)
    for k in multi:
        assert np.array_equal(multi[k], single[k]), k
    ref = ora.recognise_batch(pcm[:64], 2400, bank, T, 4096)
    assert np.array_equal(multi["score"][:64], ref["score"])
    for h in hs:
        h.close()


def test_thin_c_host_links_reference_named_symbols():
    """host/spch_host.c = save_mdl + spch_recg transcribed against the reference's headers (include/compat) and linked
    straight against libspeech_b200.so: single-call path and batched path must agree"""
    import subprocess
    exe = os.path.join(os.path.dirname(HERE), "stm32-speech-recognition_b200", "host", "spch_host")
    assert os.path.exists(exe), "host binary not built (see __graft_entry__.build)"
    r = subprocess.run([exe, "20"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0 and "0 mismatches" in r.stdout, r.stdout[-2000:]


def test_unpack12_device_expander(handle):
    rng = np.random.default_rng(12)
    for n in [2, 14, 16, 18, 4098, 1000002]:
        x = rng.integers(0, 4096, n).astype(np.uint16)
        packed, orbits = sr_b200.pack12_host(x)
        assert (orbits & 0xF000) == 0
        assert np.array_equal(handle.unpack12(packed, n), x), n


def test_packed_transport_equals_plain(handle, ora):
    """sr_recognise_batch with the 12-bit packed PCIe transport: same results as the plain transport, chunks holding a sample
    >= 4096 travel plain, and both agree with the oracle on a sample"""
    B, U, T = 9000, 8000, 7                             # 5 chunks of 2096 utterances (32 MB)
    pcm = sr_b200.synth_pcm_host(B, U, 0x7A000000)
    pcm[2500, 17] = 4096                                # chunks 1 and 4 cannot be packed
    pcm[8999, 7999] = 65535
    handle.set_bank(np.zeros((1, 4096), np.uint8), 0, 4096)
    e = handle.recognise(sr_b200.synth_pcm_host(T, U, 0x7E3A0000), 2400, want=("ftr", "status"))
    bank = sr_b200.make_bank(e["ftr"])
    handle.set_bank(bank, T, 4096)
    try:
        handle.set_transport(0)
        plain = handle.recognise(pcm, 2400)
        assert handle.transport_stats()[0] == 0
        handle.set_transport(1)
        packed = handle.recognise(pcm, 2400)
        n_packed, n_plain, nbytes = handle.transport_stats()
    finally:
        handle.set_transport(-1)
    assert n_packed + n_plain == 5 and n_plain >= 2, (n_packed, n_plain)
    cpus = len(os.sched_getaffinity(0))
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        cpus = cpus if q == "max" else min(cpus, -(-int(q) // int(per)))
    except (OSError, ValueError):
        pass
    if cpus >= 8:                                       # with fewer CPUs the library creates no packer pool: everything plain
        assert n_packed >= 1 and nbytes < pcm.nbytes, (n_packed, n_plain, nbytes)
    for k in plain:
        assert plain[k].tobytes() == packed[k].tobytes(), k
    sel = np.array([0, 2095, 2096, 2500, 4191, 4192, 8383, 8384, 8999])
    ref = ora.recognise_batch(pcm[sel], 2400, bank, T, 4096)
    _cmp_recog({k: v[sel] for k, v in packed.items()}, ref)


def test_packed_transport_under_torchrun_two_ranks():
    """the 12-bit transport with two ranks of one node sharing the CPU quota (LOCAL_WORLD_SIZE = 2: each rank sizes its
    packer pool from its share): packed == plain == device path on every rank"""
    import subprocess
    import sys
    import torch
    script = os.path.join(HERE, "_torchrun_pack.py")
    port = 29500 + (os.getpid() % 500)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), script], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert r.stdout.count("rank ok") == 2, r.stdout[-3000:]


def test_multi_gpu_c_host_nccl_allgather():
    """host/spch_host_mgpu.c: plain C + pthreads, one rank per GPU, NCCL all-gather through the C-ABI
    (sr_recognise_batch_dev_allgather); every rank's gathered scores and argmin keys == the single-GPU batch result"""
    import subprocess
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (NCCL refuses two ranks on one device)")
    exe = os.path.join(os.path.dirname(HERE), "stm32-speech-recognition_b200", "host", "spch_host_mgpu")
    assert os.path.exists(exe), "host binary not built (see __graft_entry__.build)"
    n = min(torch.cuda.device_count(), 8)
    r = subprocess.run([exe, str(n), "384"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and ": 0 mismatches" in r.stdout, r.stdout[-2000:]


def test_nccl_allgather_through_python_binding_two_ranks():
    """sr_comm_* from two processes (torchrun): the id travels through torch.distributed, the gather runs inside
    libspeech_b200.so; gathered block r on every rank == rank r's own results"""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    script = os.path.join(HERE, "_torchrun_comm.py")
    port = 29500 + ((os.getpid() + 7) % 500)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), script], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.count("rank ok") == 2, r.stdout[-3000:]


def test_numa_helpers_and_labels(handle):
    """placement helpers never fail on a single-node box and report consistently; commstr labels (main.c:25-31, 295)"""
    L = sr_b200.lib()
    node = L.sr_device_numa_node(0)
    arr, p = sr_b200.host_alloc_dev(0, 1 << 20)
    arr[:] = 7
    got = L.sr_host_numa_node(C.c_void_p(p))
    assert node < 0 or got < 0 or got == node
    sr_b200.host_free(p)
    assert handle.label(0) == b"0 " and handle.label(9) == b"9 " and handle.label(10) == bytes([0xC9, 0xCF]) and handle.label(18) is None
    h2 = sr_b200.Handle(0)
    h2.set_labels([b"on", b"off", b"up"], 4)
    assert h2.label(1) == b"off" and h2.label(3) is None
    h2.close()


def test_empty_batch_and_argument_errors(handle):
    z = np.zeros((0, 8000), np.uint16)
    assert handle.recognise(z, 2400)["cmd"].shape == (0,)
    with pytest.raises(sr_b200.SrError):
        handle.set_bank(np.zeros((2, 100), np.uint8), 2, 100)          # slot stride < sizeof(v_ftr_tag)
