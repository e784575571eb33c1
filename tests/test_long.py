"""Long-form VAD and per-segment recognition (include/sr_long.h): recordings of any length up to 2^27 samples, every
segment, one decision per segment.

CPU: the restatement sro_vad_long (tests/oracle_ext/long.c) equals a plain Python transcription of VAD.C:97-218 with the
3-segment cap removed, written here, on planted activity patterns and random PCM; its first three segments equal the port's
sro_vad and the reference's own VAD, and on any recording the segments that close before sample 65 535 equal the reference's
VAD on the first 65 535 samples (VAD is causal). A guard parses include/sr_long.h for entry points this file does not run.

GPU (bit for bit): both calls against the oracle on the reference's four digit recordings, on synthetic recordings of
ragged lengths up to 2^24 samples (poison past lens[b]), one recording of 2^27 samples, 4 096 recordings of 1-30 s, with
n_segs > max_segs and max_segs = 0, full-scale samples and threshold corners, the _dev forms at PCM 2, 6 and 14 bytes past
a 16-byte boundary; composition with the existing calls for recordings of <= 65 535 samples; real-speech decisions; threads
beside a recognise handle; and the host's group and launch plan, counted under the timing tags."""
import os
import re
import threading

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = 0xFFFFFFFF
FIXTURES = ("digits_1_10_a", "digits_1_10_b", "digits_1_9_units_a", "digits_1_9_units_b")
GROUP_BYTES = 256 << 20            # kLongGroupBytes, csrc/sr_api.cu
TAG_MFCC, TAG_STATUS, TAG_BEST_INIT, TAG_DTW, TAG_BEST_FINAL, TAG_DTW_BAND, TAG_BLOCKS, TAG_SEGS = 1, 2, 3, 4, 5, 6, 11, 12
PREFILL = 0xA5A5A5A5


# ---- the definition, transcribed: VAD.C:97-218 without max_vc_con, u32 length ----------------------------------------
def py_vad_long(vc, n, atap):
    """[(start, end)], end = NULL for a segment still open when the frames run out"""
    mid, n_thl, z_thl, s_thl = int(atap["mid_val"]), int(atap["n_thl"]), int(atap["z_thl"]), int(atap["s_thl"])
    a_thl, b_thl = (mid + n_thl) & 0xFFFFFFFF, (mid - n_thl) & 0xFFFFFFFF       # VAD.C:112-113
    vc = [int(v) for v in vc[:n]]
    last_sig, cur, front, back, segs = 0, 0, 0, 0, []
    i = 0
    while n > 160 and i < n - 160:                                               # VAD.C:121
        frm_sum = sum(abs(vc[i + h] - mid) for h in range(160))                  # VAD.C:126-129
        frm_zero = 0
        for h in range(159):                                                     # VAD.C:132-157
            if vc[i + h] >= a_thl:
                last_sig = 2
            elif vc[i + h] < b_thl:
                last_sig = 1
            w = vc[i + h + 1]
            if w >= a_thl:
                frm_zero += last_sig == 1
            elif w < b_thl:
                frm_zero += last_sig == 2
        if frm_sum > s_thl or frm_zero > z_thl:                                  # VAD.C:164-187
            if cur == 0:
                cur, front = 1, 1
            elif cur == 1:
                front += 1
                if front >= 8:
                    cur, front = 2, 0
                    segs.append([i - 7 * 80, NULL])
            elif cur == 3:
                back, cur = 0, 2
        else:                                                                    # VAD.C:188-216
            if cur == 2:
                cur, back = 3, 1
            elif cur == 3:
                back += 1
                if back >= 11:
                    cur, back = 0, 0
                    segs[-1][1] = i - 11 * 80 + 160
            elif cur == 1:
                front, cur = 0, 0
        i += 80
    return [tuple(s) for s in segs]


def _atap(mid=2048, n_thl=5000, z_thl=2, s_thl=15999):
    a = np.zeros(1, ob.ATAP_DTYPE)
    a["mid_val"], a["n_thl"], a["z_thl"], a["s_thl"] = mid, n_thl, z_thl, s_thl
    return a


def planted(runs, first_loud=True):
    """PCM whose frame k is active exactly when blocks k and k+1 are both loud, under _atap(): every sample is below
    b_thl (mid - n_thl wraps), so no band crossing counts, and a loud block sums |x - mid| = 8 000 against s_thl = 15 999.
    runs: alternating numbers of loud / quiet 80-sample blocks. A run of r active frames is r + 1 loud blocks, a run of r
    inactive frames between active ones is r - 1 quiet blocks."""
    out, loud = [], first_loud
    for r in runs:
        out.append(np.full(80 * r, 2148 if loud else 2048, np.uint16))
        loud = not loud
    return np.concatenate(out)


def _check_vad_long(lo, pcm, atap, n=None):
    n = len(pcm) if n is None else n
    want = py_vad_long(pcm, n, atap[0])
    cnt, seg = lo.vad_long(pcm[None, :n], atap, len(want) + 2)
    assert int(cnt[0]) == len(want)
    assert [tuple(s) for s in seg[0, :len(want)].tolist()] == want
    return want


def test_vad_long_equals_python_transcription_on_planted_patterns():
    lo = ox.long_oracle()
    a = _atap()
    cases = {                                            # (runs of loud / quiet blocks, first run loud)
        "8 active frames open, 7 do not": ([8, 20, 9, 20], True),
        "11 inactive frames close, 10 do not": ([9, 9, 9, 10, 9, 30], True),
        "segments back to back": ([9, 10] * 12 + [2], True),
        "open at sample 0, closed at the end": ([12, 12, 1], True),
        "open at the last frame": ([30, 10], False),
        "open when the frames run out": ([4, 30, 40], True),
        "exactly 160 samples, no frame": ([2], False),
    }
    got = {name: _check_vad_long(lo, planted(runs, first), a) for name, (runs, first) in cases.items()}
    _check_vad_long(lo, np.full(161, 2148, np.uint16), a)                # 161 samples: one frame
    assert got["8 active frames open, 7 do not"] == [(28 * 80, 36 * 80 + 80)]   # blocks 28..36 loud: frames 28..35
    assert got["11 inactive frames close, 10 do not"] == [(0, 2160), (2960, 3680)]
    assert len(got["segments back to back"]) == 12 and all(e != NULL for _, e in got["segments back to back"])
    assert got["open at sample 0, closed at the end"] == [(0, 11 * 80 + 80)]
    assert got["open at the last frame"] == [(30 * 80, NULL)]
    assert got["open when the frames run out"][-1][1] == NULL
    assert got["exactly 160 samples, no frame"] == []


def test_vad_long_thousands_of_segments():
    lo = ox.long_oracle()
    rng = np.random.default_rng(1)
    runs = []
    for _ in range(2000):
        runs += [int(rng.integers(8, 12)), int(rng.integers(9, 13))]
    pcm = planted(runs)
    want = _check_vad_long(lo, pcm, _atap())
    assert len(want) >= 1000


def test_vad_long_equals_python_transcription_on_random_pcm():
    lo = ox.long_oracle()
    rng = np.random.default_rng(2)
    for t in range(12):
        n = int(rng.integers(100, 12000))
        # bursts of loud, band-crossing noise on a quiet floor
        pcm = (2048 + rng.integers(-20, 21, n)).astype(np.int64)
        for _ in range(int(rng.integers(0, 8))):
            s = int(rng.integers(0, n))
            e = min(n, s + int(rng.integers(200, 2500)))
            pcm[s:e] += rng.integers(-900, 901, e - s)
        pcm = np.clip(pcm, 0, 4095).astype(np.uint16)
        a = _atap(2048, int(rng.integers(10, 60)), 2, int(rng.integers(500, 4000)))
        _check_vad_long(lo, pcm, a)


def test_first_three_segments_equal_vad_and_reference():
    lo, port = ox.long_oracle(), ob.port()
    ref = ob.ref() if ob.have_ref() else None
    recs = [ox.golden_wav(f)[:65535] for f in FIXTURES] + list(sr_b200.synth_pcm_host(6, 40000, 0x10E6, 6))
    recs.append(ox.synth_long(1, 65535, 0x10E7)[0])
    for pcm in recs:
        n = len(pcm)
        a = port.noise_atap(pcm, 2400)
        cnt, seg = lo.vad_long(pcm[None], a, 64)
        three = port.vad(pcm, n, a)
        k = min(int(cnt[0]), 3)
        got = np.full(6, NULL, np.uint32)
        got[:2 * k] = seg[0, :k].reshape(-1)
        assert got.tolist() == three.tolist(), (got, three)
        if ref is not None:
            assert ref.vad(pcm, n, a).tolist() == three.tolist()


def test_segments_closing_before_65535_equal_reference_vad():
    """VAD is causal: on any recording, the long-form segments that close before sample 65 535 are the reference's VAD on
    the first 65 535 samples, up to its three segments"""
    lo, port = ox.long_oracle(), ob.port()
    vad65 = (ob.ref() if ob.have_ref() else port).vad
    recs = [ox.golden_wav(f) for f in FIXTURES] + list(ox.synth_long(3, 300000, 0x10E8))
    for pcm in recs:
        a = port.noise_atap(pcm, 2400)
        cnt, seg = lo.vad_long(pcm[None], a, 256)
        # a segment closes at frame i = end + 11*80 - 160 (VAD.C:201), and the prefix has the frames i < 65535 - 160
        closed = [tuple(s) for s in seg[0, :int(cnt[0])].tolist() if s[1] != NULL and s[1] + 720 < 65535 - 160]
        three = vad65(pcm[:65535], 65535, a).reshape(3, 2).tolist()
        assert [tuple(s) for s in three if s[1] != NULL] == closed[:3]


# ---- the header guard ------------------------------------------------------------------------------------------------
def test_every_long_entry_point_is_run_here():
    """every sr_* entry point of include/sr_long.h is exercised by a GPU test of this file"""
    hdr = open(os.path.join(ROOT, "include", "sr_long.h")).read()
    names = set(re.findall(r"\bint\s+(sr_\w+)\s*\(", hdr))
    assert names == {"sr_vad_long_batch", "sr_recognise_long_batch", "sr_vad_long_batch_dev", "sr_recognise_long_batch_dev"}
    src = open(os.path.abspath(__file__)).read()
    py = {"sr_vad_long_batch": ".vad_long_batch(", "sr_recognise_long_batch": ".recognise_long_batch(",
          "sr_vad_long_batch_dev": ".vad_long_batch_dev(", "sr_recognise_long_batch_dev": ".recognise_long_batch_dev("}
    for n in names:
        assert src.count(py[n]) >= 2, n                  # in a correctness test and in the concurrency test


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _bank_of(ftr, valid_slots=None):
    """one template per feature struct, template k in slot 4k (cmd = k); the other slots erased"""
    K = len(ftr)
    ftr4 = np.zeros(4 * K, ob.FTR_DTYPE)
    ftr4[0::4] = ftr
    valid = np.zeros(4 * K, bool)
    valid[0::4] = True
    return sr_b200.make_bank(ftr4, 4096, valid), 4 * K


def _cmp_recognise(got, want, rows=None):
    rows = range(len(want["n_segs"])) if rows is None else rows
    for b in rows:
        assert got["n_segs"][b] == want["n_segs"][b], b
        assert got["atap"][b].tobytes() == want["atap"][b].tobytes(), b
        m = min(int(want["n_segs"][b]), got["segs"].shape[1])
        assert got["segs"][b, :m].tobytes() == want["segs"][b, :m].tobytes(), (b, got["segs"][b, :m], want["segs"][b, :m])


@pytest.mark.gpu
def test_fixtures_bit_exact(handle):
    lo, port = ox.long_oracle(), ob.port()
    recs = [ox.golden_wav(f) for f in FIXTURES]
    U = max(len(r) for r in recs)
    pcm = np.zeros((4, U), np.uint16)
    lens = np.array([len(r) for r in recs], np.uint32)
    for b, r in enumerate(recs):
        pcm[b, :len(r)] = r
        pcm[b, len(r):] = 4095                                   # poison past lens[b]
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    v = handle.vad_long_batch(pcm, 32, 2400, lens)
    n, seg = lo.vad_long(pcm, v["atap"], 32, lens)
    assert v["n_segs"].tolist() == n.tolist() and (v["seg_off"] == seg).all()
    assert v["n_segs"].tolist() == [10, 10, 13, 13], v["n_segs"]
    got = handle.recognise_long_batch(pcm, 32, 2400, lens)
    _cmp_recognise(got, ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 32, lens))


def _synth_long(lengths, U, seed):
    """recordings of the given lengths (many words each) in rows of U samples, poisoned past their length"""
    pcm = ox.synth_long(len(lengths), U, seed)
    for b, n in enumerate(lengths):
        pcm[b, n:] = np.where(np.arange(U - n) % 2, 4095, 0)
    return pcm


@pytest.mark.gpu
def test_ragged_synthetic_lengths(handle):
    lo, port = ox.long_oracle(), ob.port()
    lens = np.array([160, 161, 240, 65535, 65536, 1000003, 1 << 24], np.uint32)
    pcm = _synth_long(lens, 1 << 24, 0x10A0)
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    for geom in (0, 1):
        handle.set_geometry(geom)
        got = handle.recognise_long_batch(pcm, 4096, 2400, lens)
        want = ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 4096, lens, geom_b=geom == 1)
        _cmp_recognise(got, want)
    handle.set_geometry(0)
    assert int(got["n_segs"][-1]) > 1000


@pytest.mark.gpu
def test_one_recording_of_2_27_samples(handle):
    lo = ox.long_oracle()
    U = 1 << 27
    pcm = ox.synth_long(1, U, 0x10B0)
    v = handle.vad_long_batch(pcm, 40000, 2400)
    n, seg = lo.vad_long(pcm, v["atap"], 40000)
    assert int(v["n_segs"][0]) == int(n[0]) > 1000
    assert (v["seg_off"] == seg).all()


@pytest.mark.gpu
def test_4096_recordings_of_1_to_30_s(handle):
    lo, port = ox.long_oracle(), ob.port()
    rng = np.random.default_rng(4)
    B, U = 4096, 240000
    lens = rng.integers(8000, U + 1, B).astype(np.uint32)
    pcm = ox.synth_long(B, U, 0x10C0)
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    got = handle.recognise_long_batch(pcm, 64, 2400, lens)
    atap = ox.atap_long(port, pcm, 2400, lens)
    n, seg = lo.vad_long(pcm, atap, 64, lens)
    assert got["n_segs"].tolist() == n.tolist()
    assert (got["segs"]["start"] == np.where(np.arange(64)[None] < n[:, None], seg[..., 0], 0)).all()
    rows = sorted({0, B - 1, *rng.integers(0, B, 14).tolist()})
    _cmp_recognise(got, ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 64, lens, rows=rows), rows)


@pytest.mark.gpu
def test_max_segs_cuts_and_prefilled_outputs(handle):
    lo, port = ox.long_oracle(), ob.port()
    pcm = ox.synth_long(3, 200000, 0x10D0)
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    full = ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 64)
    assert (full["n_segs"] > 3).all()
    for ms in (0, 1, 3):
        segs = np.zeros((3, ms), ox.LONG_SEG_DTYPE)
        segs.view(np.uint32)[...] = PREFILL
        got = handle.recognise_long_batch(pcm, ms, 2400, segs=segs)
        assert got["n_segs"].tolist() == full["n_segs"].tolist()
        assert got["segs"].tobytes() == full["segs"][:, :ms].tobytes()
        seg_off = np.full((3, ms, 2), PREFILL, np.uint32)
        v = handle.vad_long_batch(pcm, ms, 2400, seg_off=seg_off)
        assert v["n_segs"].tolist() == full["n_segs"].tolist()
        assert (v["seg_off"][..., 0] == full["segs"]["start"][:, :ms]).all()
    # records past n_segs keep the caller's bytes
    segs = np.zeros((3, 64), ox.LONG_SEG_DTYPE)
    segs.view(np.uint32)[...] = PREFILL
    got = handle.recognise_long_batch(pcm, 64, 2400, segs=segs)
    for b in range(3):
        assert (got["segs"][b, int(got["n_segs"][b]):].view(np.uint32) == PREFILL).all()


@pytest.mark.gpu
def test_full_scale_samples_and_threshold_corners(handle):
    lo = ox.long_oracle()
    rng = np.random.default_rng(5)
    U = 150000
    pcm = rng.integers(0, 65536, (6, U)).astype(np.uint16)
    pcm[1] = np.where(rng.random(U) < 0.5, 0, 65535)
    pcm[2, ::3] = 32768
    corners = [(0, 0, 0, 0), (65535, 65535, 65535, 0xFFFFFFFF), (70000, 1000, 2, 4000000), (32768, 0, 2, 5000000),
               (32768, 32768, 2, 5000000), (1, 2, 0, 0)]
    atap = np.zeros(6, ob.ATAP_DTYPE)
    for b, (m, n_thl, z, s) in enumerate(corners):
        atap[b] = (m, n_thl, z, s)
    v = handle.vad_long_batch(pcm, 4096, 0, atap=atap.copy())           # n_len = 0: noise_atap leaves atap as passed
    assert v["atap"].tobytes() == atap.tobytes()
    n, seg = lo.vad_long(pcm, atap, 4096)
    assert v["n_segs"].tolist() == n.tolist() and (v["seg_off"] == seg).all()
    # noise_atap on full-scale samples
    v = handle.vad_long_batch(pcm, 4096, 2400)
    assert v["atap"].tobytes() == ox.atap_long(ob.port(), pcm, 2400).tobytes()
    n, seg = lo.vad_long(pcm, v["atap"], 4096)
    assert v["n_segs"].tolist() == n.tolist() and (v["seg_off"] == seg).all()


@pytest.mark.gpu
def test_dev_forms_at_unaligned_pcm(handle):
    import torch
    lo, port = ox.long_oracle(), ob.port()
    lens = np.array([70001, 161, 123457, 99999], np.uint32)
    U = 123457
    pcm = _synth_long(lens, U, 0x10E0)
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    want = ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 40, lens)
    dev = torch.device("cuda:0")
    for off in (2, 6, 14):
        raw = torch.zeros(pcm.nbytes + 64, dtype=torch.uint8, device=dev)
        base = (16 - raw.data_ptr() % 16) % 16 + off
        raw[base:base + pcm.nbytes] = torch.from_numpy(pcm.view(np.uint8).reshape(-1)).to(dev)
        d_lens = torch.from_numpy(lens.view(np.int32)).to(dev)
        d_atap = torch.zeros(4 * 12, dtype=torch.uint8, device=dev)
        d_n = torch.zeros(4, dtype=torch.int32, device=dev)
        d_seg = torch.full((4 * 40 * 2,), -1, dtype=torch.int32, device=dev)
        handle.vad_long_batch_dev(raw.data_ptr() + base, U, 4, d_lens.data_ptr(), 2400, 40, d_atap.data_ptr(), d_n.data_ptr(),
                                  d_seg.data_ptr())
        d_segs = torch.zeros(4 * 40 * 7, dtype=torch.int32, device=dev)
        d_atap2 = torch.zeros(4 * 12, dtype=torch.uint8, device=dev)
        d_n2 = torch.zeros(4, dtype=torch.int32, device=dev)
        handle.recognise_long_batch_dev(raw.data_ptr() + base, U, 4, d_lens.data_ptr(), 2400, 40, d_atap2.data_ptr(),
                                        d_n2.data_ptr(), d_segs.data_ptr())
        handle.sync()
        n = d_n.cpu().numpy().view(np.uint32)
        seg = d_seg.cpu().numpy().view(np.uint32).reshape(4, 40, 2)
        assert n.tolist() == want["n_segs"].tolist()
        for b in range(4):
            m = min(int(n[b]), 40)
            assert (seg[b, :m, 0] == want["segs"]["start"][b, :m]).all() and (seg[b, :m, 1] == want["segs"]["end"][b, :m]).all()
        got = dict(atap=d_atap2.cpu().numpy().view(ob.ATAP_DTYPE), n_segs=d_n2.cpu().numpy().view(np.uint32),
                   segs=d_segs.cpu().numpy().view(ox.LONG_SEG_DTYPE).reshape(4, 40))
        _cmp_recognise(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [0, 1])
def test_composition_with_the_existing_calls(handle, geom):
    """for recordings of <= 65 535 samples: records 0-2 = sr_vad_batch, segment 0 = sr_recognise_batch, every segment =
    sr_mfcc_batch + sr_dtw_batch on its (row, segment), under the greedy walk and r in {10, 15, 118}"""
    B, U = 24, 65535
    pcm = ox.synth_long(B, U, 0x10F0 + geom)
    bank, T = ox.synth_bank()
    handle.set_bank(bank, T, 4096)
    handle.set_geometry(geom)
    try:
        for flags, r in ((0, 0), (2, 10), (2, 15), (2, 118)):
            handle.set_match(flags, r)
            got = handle.recognise_long_batch(pcm, 32, 2400)
            v = handle.vad_long_batch(pcm, 32, 2400)
            three = handle.vad(pcm, v["atap"])
            rec = handle.recognise(pcm, 2400)
            for b in range(B):
                k = min(int(v["n_segs"][b]), 3)
                want = np.full(6, NULL, np.uint32)
                want[:2 * k] = v["seg_off"][b, :k].reshape(-1)
                assert three[b].reshape(-1).tolist() == want.tolist()
                s0 = got["segs"][b, 0]
                if v["n_segs"][b]:
                    assert (s0["status"], s0["best_idx"], s0["best_dis"], s0["cmd"]) == \
                        (rec["status"][b], rec["best_idx"][b], rec["best_dis"][b], rec["cmd"][b])
            # every segment through sr_mfcc_batch + sr_dtw_batch on its own row
            rows, segs = [], []
            for b in range(B):
                for k in range(min(int(got["n_segs"][b]), 32)):
                    rows.append(b)
                    segs.append(v["seg_off"][b, k])
            sel = pcm[rows]
            ftr = handle.mfcc(sel, np.array(segs, np.uint32), v["atap"][rows])
            score, bi, bd = handle.dtw(ftr, 1 | flags, r)
            recs = np.concatenate([got["segs"][b, :min(int(got["n_segs"][b]), 32)] for b in range(B)])
            ok = recs["status"] == 0
            assert (recs["frm_num"][recs["end"] != NULL] == ftr["frm_num"][recs["end"] != NULL]).all()
            assert (recs["best_idx"][ok] == bi[ok]).all() and (recs["best_dis"][ok] == bd[ok]).all()
    finally:
        handle.set_match(0, 0)
        handle.set_geometry(0)


@pytest.mark.gpu
def test_real_speech_decisions():
    """enrol one digit recording's segments (template k in slot 4k) and recognise the other, both directions, both pairs:
    GPU decisions equal the oracle's. Accuracy is reported (DESIGN.md), not asserted."""
    lo, port = ox.long_oracle(), ob.port()
    h = sr_b200.Handle(0)
    try:
        for a_name, b_name in ((FIXTURES[0], FIXTURES[1]), (FIXTURES[1], FIXTURES[0]), (FIXTURES[2], FIXTURES[3]),
                               (FIXTURES[3], FIXTURES[2])):
            a, b = ox.golden_wav(a_name), ox.golden_wav(b_name)
            for flags, r in ((0, 0), (2, 118)):
                h.set_match(flags, r)
                h.set_bank(np.zeros((0, 4096), np.uint8), 0, 4096)
                ea = h.recognise_long_batch(a[None], 32, 2400)
                ma = int(ea["n_segs"][0])
                at = ea["atap"]
                ftr = ox.ftr_of_segments(port, a[None], at, [(0, int(s["start"]), int(s["end"]) if s["end"] != NULL else int(s["start"]))
                                                             for s in ea["segs"][0, :ma]])
                bank, T = _bank_of(ftr)
                h.set_bank(bank, T, 4096)
                got = h.recognise_long_batch(b[None], 32, 2400)
                want = ox.recognise_long(lo, port, b[None], 2400, bank, T, 4096, 32, band_r=-1 if flags == 0 else r)
                _cmp_recognise(got, want)
                m = min(int(got["n_segs"][0]), ma)
                right = int((got["segs"][0, :m]["cmd"] == np.arange(m)).sum())
                print("%s -> %s, %s: %d/%d" % (a_name, b_name, "greedy" if flags == 0 else "r=%d" % r, right, m))
    finally:
        h.close()


# ---- concurrency ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_threads_beside_a_recognise_handle():
    import torch
    lens = np.array([90000, 150000, 40000], np.uint32)
    pcm = _synth_long(lens, 150000, 0x1100)
    short = sr_b200.synth_pcm_host(64, 16000, 0x1110, 3)
    bank, T = ox.synth_bank()
    dev = torch.device("cuda:0")

    def job_vad(h):
        return h.vad_long_batch(pcm, 32, 2400, lens)

    def job_rec(h):
        return h.recognise_long_batch(pcm, 32, 2400, lens)

    def job_dev(h):
        d_pcm = torch.from_numpy(pcm.view(np.int16)).to(dev)
        d_lens = torch.from_numpy(lens.view(np.int32)).to(dev)
        d_atap = torch.zeros(3 * 12, dtype=torch.uint8, device=dev)
        d_n, d_n2 = torch.zeros(3, dtype=torch.int32, device=dev), torch.zeros(3, dtype=torch.int32, device=dev)
        d_seg = torch.zeros(3 * 32 * 2, dtype=torch.int32, device=dev)
        d_rec = torch.zeros(3 * 32 * 7, dtype=torch.int32, device=dev)
        h.vad_long_batch_dev(d_pcm.data_ptr(), 150000, 3, d_lens.data_ptr(), 2400, 32, d_atap.data_ptr(), d_n.data_ptr(),
                             d_seg.data_ptr())
        h.recognise_long_batch_dev(d_pcm.data_ptr(), 150000, 3, d_lens.data_ptr(), 2400, 32, None, d_n2.data_ptr(),
                                   d_rec.data_ptr())
        h.sync()
        return dict(n=d_n.cpu().numpy(), seg=d_seg.cpu().numpy(), n2=d_n2.cpu().numpy(), rec=d_rec.cpu().numpy())

    def job_short(h):
        return h.recognise(short, 2400)

    jobs = [job_vad, job_rec, job_dev, job_short]
    handles = [sr_b200.Handle(0) for _ in jobs]
    try:
        for h in handles:
            h.set_bank(bank, T, 4096)
        serial = [j(h) for j, h in zip(jobs, handles)]
        results = [[None] * 3 for _ in jobs]
        errors = []

        def run(i):
            try:
                for rep in range(3):
                    results[i][rep] = jobs[i](handles[i])
            except Exception as e:                      # noqa: BLE001
                errors.append(e)
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        for i in range(len(jobs)):
            for rep in range(3):
                for k, v in serial[i].items():
                    assert np.asarray(results[i][rep][k]).tobytes() == np.asarray(v).tobytes(), (jobs[i].__name__, k)
    finally:
        for h in handles:
            h.close()


# ---- the host's plan, counted -------------------------------------------------------------------------------------------
def _tags(h):
    t = [tag for tag, _ in h.timing_collect()]
    return {k: t.count(k) for k in set(t)}


@pytest.mark.gpu
def test_groups_and_launches_are_counted():
    """groups of at most 256 MB of PCM (at least one recording), 3 VAD launches per group (tags 11, 11, 12) and, for
    recognition, 7 more (flat table 2 untimed, get_mfcc, status, best-init, scan, scatter); the segment count of a group
    past one grid pass of every recognition kernel"""
    lo, port = ox.long_oracle(), ob.port()
    h = sr_b200.Handle(0)
    try:
        bank, T = ox.synth_bank()
        h.set_bank(bank, T, 4096)
        h.timing_enable(4096)
        U = 1 << 24
        lens = np.array([U, U - 7, 3 * 80000, U, 161, U, U - 1, U, 999999, U, U], np.uint32)
        pcm = _synth_long(lens, U, 0x1200)
        G = max(1, GROUP_BYTES // (2 * U))
        groups = -(-len(lens) // G)
        assert G == 8 and groups == 2
        c0 = h.launch_count()
        got = h.recognise_long_batch(pcm, 4096, 2400, lens)
        assert h.launch_count() - c0 == 10 * groups
        assert _tags(h) == {TAG_BLOCKS: 2 * groups, TAG_SEGS: groups, TAG_MFCC: groups, TAG_STATUS: groups,
                            TAG_BEST_INIT: groups, TAG_DTW: groups, TAG_BEST_FINAL: groups}
        assert int(got["n_segs"][:G].sum()) > 132 * 4 and int(got["n_segs"][G:].sum()) > 132
        rows = [0, G - 1, G, len(lens) - 1, 4]
        _cmp_recognise(got, ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 4096, lens, rows=rows), rows)
        # the same recordings one group at a time
        for g0 in range(0, len(lens), G):
            part = h.recognise_long_batch(pcm[g0:g0 + G], 4096, 2400, lens[g0:g0 + G])
            for k in ("atap", "n_segs", "segs"):
                assert part[k].tobytes() == got[k][g0:g0 + G].tobytes(), k
        h.timing_collect()
        c0 = h.launch_count()
        h.vad_long_batch(pcm, 0, 2400, lens)
        assert h.launch_count() - c0 == 3 * groups
        assert _tags(h) == {TAG_BLOCKS: 2 * groups, TAG_SEGS: groups}
        c0 = h.launch_count()
        h.recognise_long_batch(pcm[:2], 0, 2400, lens[:2])                # max_segs = 0 counts only
        assert h.launch_count() - c0 == 3
    finally:
        h.close()
