"""The banded dynamic-programming matcher (K3, an extension the reference does not have; parity unpinned) at every radius
up to the full matrix, and as the matcher of the recognition paths (sr_set_match).

CPU: the oracle's sro_dtw_band equals the plain band_dp_ref of refs.py at the wide radii, and the textbook
full_dp_ref where the band covers every column. GPU: sr_dtw_batch with SR_DTW_BAND equals the oracle at those radii (the
whole-row kernel for r >= 16); recognition, streaming and the multi-handle call under the band matcher equal the oracle's
own composition of the same stages. Every GPU test makes its own handles, so the session handle never carries a matcher."""
import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from cases import band_cases, band_rows, guard_edge_shapes, make_ftr
from drive import handle, recognise_dev_np, same
from refs import DIS_ERR, MAX_FRM, NTHREADS, band_dp_ref, full_dp_ref

WIDE_RADII = (16, 31, 32, 59, 117, 118, 119, 1000)
INT32_MAX = 2 ** 31 - 1
STRIDE = ob.FTR_DTYPE.itemsize
BAND = sr_b200.DTW_BAND
# tags of sr_timing_collect
VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL, DTW_BAND = range(7)


# ---- the oracle at the wide radii (CPU) ---------------------------------------------------------------------------
def test_dtw_band_oracle_equals_plain_references_at_wide_radii():
    """sro_dtw_band == band_dp_ref for r in {16, 31, 32, 59, 117, 118, 119, 1000} on every (I, M) of the 2:1 guard's edges
    and the corners, with small, +-32 767 and all-equal rows; where the band covers every column (r >= M - 1, so every
    r >= 118) it also equals the textbook full_dp_ref. band_dp_ref is evaluated once per distinct band: r and min(r, M - 1)
    select the same cells, as |j - floor(i*M/I)| <= M - 1 for every column j"""
    po = ob.port()
    rng = np.random.default_rng(0xD9)
    kinds = ("small", "full", "equal")
    n_full = n_narrow = 0
    for k, (I, M) in enumerate(guard_edge_shapes()):
        fin, fmdl = band_rows(rng, I, kinds[k % 3]), band_rows(rng, M, kinds[k % 3])
        fi, fm = make_ftr([fin]), make_ftr([fmdl])
        got = {r: int(po.dtw_batch(fi, fm.view(np.uint8), 1, STRIDE, band_r=r)[0][0, 0]) for r in WIDE_RADII}
        want = {}
        for r in WIDE_RADII:
            eff = min(r, M - 1)
            if eff not in want:
                want[eff] = band_dp_ref(fin, fmdl, eff)
            assert got[r] == want[eff], (I, M, kinds[k % 3], r, got[r], want[eff])
            n_narrow += r < M - 1
        full = full_dp_ref(fin, fmdl)
        for r in WIDE_RADII:
            if r >= min(MAX_FRM - 1, M - 1):
                assert got[r] == full, (I, M, r)
                n_full += 1
    assert n_full > 1000 and n_narrow > 300


# ---- sr_dtw_batch at the wide radii (GPU) --------------------------------------------------------------------------
@pytest.mark.gpu
def test_dtw_batch_wide_band_equals_oracle_on_every_shape():
    """sr_dtw_batch with SR_DTW_BAND at r in {16, 31, 32, 59, 117, 118, 119, 1000, INT32_MAX}: score, best_idx and best_dis
    bit for bit against the oracle on every pair of the four 119 x 119 cases of test_extension_refs (INT32_MAX against
    the r = 118 result: the oracle's c + r would overflow), against band_dp_ref / full_dp_ref on a sample, the largest
    local distance on every cell of the 60- and 119-row sets, self-matches 0. A wider band never raises a score."""
    po = ob.port()
    rng = np.random.default_rng(0x3D)
    h = sr_b200.Handle(0)
    n_checked = 0
    for name, utt, tpl in band_cases():
        fin, bank = make_ftr(utt), make_ftr(tpl)
        T = len(bank)
        I = fin["frm_num"].astype(np.int64)[:, None]
        M = bank["frm_num"].astype(np.int64)[None, :]
        walks = (I <= 2 * M) & (M <= 2 * I)
        h.set_bank(bank.view(np.uint8).reshape(T, STRIDE), T, STRIDE)
        scores = {}
        for r in WIDE_RADII + (INT32_MAX,):
            score, bi, bd = h.dtw(fin, flags=sr_b200.DTW_BAND, band_r=r)
            want = scores[118] if r == INT32_MAX else po.dtw_batch(fin, bank.view(np.uint8), T, STRIDE, band_r=r,
                                                                     nthreads=NTHREADS)[0]
            assert np.array_equal(score, want), (name, r)
            key = (want.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
            kmin = key.min(axis=1)
            assert np.array_equal(bi, (kmin & np.uint64(0xFFFFFFFF)).astype(np.uint32)), (name, r)
            assert np.array_equal(bd, (kmin >> np.uint64(32)).astype(np.uint32)), (name, r)
            pairs = [(118, 118), (59, 118), (118, 59), (0, 0), (0, 1), (1, 0)] + [tuple(rng.choice(np.argwhere(walks)))]
            for u, t in pairs:
                want_ut = band_dp_ref(utt[u], tpl[t], min(r, MAX_FRM - 1))
                assert score[u, t] == want_ut, (name, r, u, t)
                if r >= MAX_FRM - 1:
                    assert score[u, t] == full_dp_ref(utt[u], tpl[t]), (name, r, u, t)
                n_checked += 1
            assert (score[~walks] == DIS_ERR).all() and (score[walks] != DIS_ERR).all(), (name, r)   # 2r+1 >= 33 > any shift
            if name == "self":
                assert (np.diag(score) == 0).all()
            if name == "equal":
                assert (score == np.where(walks, 0, DIS_ERR)).all()
            if name == "full":                   # max(I, M) cells of 65 536 on the cheapest path
                assert score[118, 118] == 119 * 65536 // 238 and score[118, 59] == 119 * 65536 // 179
                assert score[59, 118] == 119 * 65536 // 179 and score[59, 59] == 60 * 65536 // 120
            scores[r] = score
        S = np.stack([scores[r] for r in WIDE_RADII]).astype(np.int64)
        assert (S[1:] <= S[:-1]).all(), name
        assert np.array_equal(scores[INT32_MAX], scores[1000])
    h.close()
    assert n_checked == 4 * 9 * 7


# ---- recognition under the band matcher ----------------------------------------------------------------------------
RADII = (0, 7, 10, 15, 16, 118)          # both sides of the kernel choice: thread form (10), warp-scan (<= 15), whole row
U = 16000
PLANTED = [0, 1, 1047, 1048, 1049, 2096, 2500, 3199]     # segments from sample 0, at and next to the 1 048-utterance chunks


def _bank(ora, slots, valid):
    """flash-layout bank of the given template indices (duplicates tie), with unsigned slots where valid is 0. The eight
    templates include two short ones whose segment starts at sample 0, so planted utterances pass the 2:1 guard"""
    tpl = sr_b200.synth_pcm_host(8, 8000, 0x7E3A0000)
    ob.plant_sample0(tpl, [1, 4], 0x7E3A)
    e = ob.recognise_pinned(ora, tpl, 2400, None, 0, 4096)
    assert (e["status"] == 0).all()
    return sr_b200.make_bank(e["ftr"][slots], valid=valid)


@pytest.fixture(scope="module")
def recog_case():
    """3 200 two-second utterances (four 1 048-utterance chunks of the host call, so the packed transport engages):
    a silent one (VAD fails), one whose word is longer than 119 frames (MFCC fails), planted segments from sample 0;
    the front end once, from the oracle's stages (recognise_pinned); a 20-slot bank with duplicates and unsigned slots
    and a 70-slot one (wider than a tile: the bank order is active)"""
    ora = ob.best_oracle()
    B = 3200
    pcm = sr_b200.synth_pcm_host(B, U, 0xD7D70000, 2)
    rng = np.random.default_rng(0xD7)
    pcm[3] = 2048
    pcm[4, 3000:13500] = 2048 + (1200 * np.sin(np.arange(10500) * 0.3)).astype(np.int64) + rng.integers(-50, 50, 10500)
    ob.plant_sample0(pcm, PLANTED, 0xD7)
    front = ob.recognise_pinned(ora, pcm, 2400, None, 0, 4096)
    assert front["status"][3] == 1 and front["status"][4] == 2
    assert (front["seg_off"][PLANTED, 0, 0] == 0).all() and (front["status"][PLANTED] == 0).all()
    base = list(range(8))
    slots20 = base + [0, 2, 5, 5, 1, 7, 3, 3, 6, 4, 0, 2]
    valid20 = [1] * 20
    valid20[3] = valid20[9] = 0
    slots70 = [int(x) for x in rng.integers(0, 8, 70)]
    valid70 = [int(x) for x in rng.integers(0, 8, 70) != 0]
    return {"pcm": pcm, "front": front, "bank20": _bank(ora, slots20, valid20), "bank70": _bank(ora, slots70, valid70)}


@pytest.mark.gpu
@pytest.mark.parametrize("r", RADII)
def test_recognise_band_matcher_equals_oracle_composition(recog_case, r):
    """set_match(SR_DTW_BAND, r): the host call on the plain and on the packed transport, one sr_recognise_batch_dev
    launch and sr_recognise_batch_multi over three handles on one GPU all equal the oracle composition, every field; with
    VAD and MFCC failures, unsigned slots, duplicate templates (ties), utterances whose segment starts at sample 0, and a
    70-slot bank (bank order active)"""
    pcm, front = recog_case["pcm"], recog_case["front"]
    bank = recog_case["bank20"]
    want = ox.compose_recognise(front, bank, 20, BAND, r)
    assert (want["best_dis"][want["status"] == 0] != ob.NULL).sum() > 2000
    h = handle(bank, 20, BAND, r)
    assert h.match() == (sr_b200.DTW_BAND, r)
    h.set_transport(0)
    same(h.recognise(pcm, 2400), want, "host plain")
    assert h.transport_stats()[:2] == (0, 4)
    h.set_transport(1)
    same(h.recognise(pcm, 2400), want, "host packed")
    assert h.transport_stats()[0] > 0
    same(recognise_dev_np(h, pcm, 2400, 20), want, "device launch")
    h.use_own_stream()
    hs = [h] + [handle(bank, 20, BAND, r) for _ in range(2)]
    same(sr_b200.recognise_multi(hs, pcm, 2400, want=sr_b200.RECOG_FIELDS), want, "multi")
    for x in hs:
        x.close()
    h70 = handle(recog_case["bank70"], 70, BAND, r)
    n = 640
    same(h70.recognise(pcm[:n], 2400),
         ox.compose_recognise({k: v[:n] for k, v in front.items()}, recog_case["bank70"], 70, BAND, r), "70-slot bank")
    h70.close()


@pytest.mark.gpu
def test_band_matcher_setting_and_greedy_round_trip(recog_case):
    """a fresh handle reports the greedy walk; negative radii and unknown flag bits fail and leave the setting alone;
    switching to the band and back reproduces the greedy results bit for bit, and the greedy results are the oracle's
    greedy composition"""
    pcm = recog_case["pcm"][:512]
    bank = recog_case["bank20"]
    h = sr_b200.Handle(0)
    h.set_bank(bank, 20, 4096)
    assert h.match() == (0, 0)
    greedy = h.recognise(pcm, 2400)
    want = ob.recognise_pinned(ob.best_oracle(), pcm, 2400, bank, 20, 4096)
    same(greedy, want, "greedy")
    for flags, r in ((sr_b200.DTW_BAND, -1), (sr_b200.DTW_CHECK_SIGN, 0), (sr_b200.DTW_BAND | 4, 3), (8, 0), (0, -5)):
        with pytest.raises(sr_b200.SrError):
            h.set_match(flags, r)
        assert h.match() == (0, 0)
    h.set_match(sr_b200.DTW_BAND, 16)
    band = h.recognise(pcm, 2400)
    assert h.match() == (sr_b200.DTW_BAND, 16)
    assert not np.array_equal(band["score"], greedy["score"])
    h.set_match(0, 0)
    again = h.recognise(pcm, 2400)
    for k in sr_b200.RECOG_FIELDS:
        assert again[k].tobytes() == greedy[k].tobytes(), k
    h.close()


@pytest.mark.gpu
def test_band_matcher_recognise_launches_are_tagged_dtw_band(recog_case):
    """timed recognise launches carry tag 6 for the band kernel at every kernel choice (r = 10, 15, 16, 118), tag 4 under
    the greedy walk"""
    pcm = recog_case["pcm"][:64]
    h = handle(recog_case["bank20"], 20)
    h.set_transport(0)
    h.timing_enable(64)
    h.recognise(pcm, 2400)
    assert [t for t, _ in h.timing_collect()] == [VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL]
    for r in (10, 15, 16, 118):
        h.set_match(sr_b200.DTW_BAND, r)
        h.recognise(pcm, 2400)
        assert [t for t, _ in h.timing_collect()] == [VAD_, MFCC_, STATUS, BEST_INIT, DTW_BAND, BEST_FINAL], r
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("r", (10, 16))
def test_geom_b_recognise_band_matcher_equals_own_oracle(r):
    """GEOM_B features (parity unpinned) under the band matcher: the port's GEOM_B front end, then its banded dtw"""
    po = ob.port()
    h = sr_b200.Handle(0)
    h.set_geometry(1)
    T = 6
    bank, est = h.enrol(sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000), 2400)
    assert (est == 0).all()
    h.set_bank(bank, T, 4096)
    h.set_match(sr_b200.DTW_BAND, r)
    pcm = sr_b200.synth_pcm_host(128, 8000, 0x5EED0000)
    ob.plant_sample0(pcm, [0, 5, 127], 0xB5)
    front = ob.recognise_pinned(po, pcm, 2400, None, 0, 4096, geom_b=True)
    want = ox.compose_recognise(front, bank, T, BAND, r)
    same(h.recognise(pcm, 2400), want, "GEOM_B")
    assert (want["status"] == 0).sum() > 100
    h.close()


# ---- streaming under the band matcher ------------------------------------------------------------------------------
def _stream_events(pool, pcm, arrival, rng):
    S, L = pcm.shape
    events = []
    if arrival == "lockstep":
        for n0 in range(0, L, 800):
            events += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 800]))
        return events
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
    return events


@pytest.mark.gpu
@pytest.mark.parametrize("arrival,group", [("lockstep", False), ("ragged", False), ("ragged", True)],
                         ids=["lockstep", "ragged", "group_of_two"])
def test_streaming_band_matcher_equals_batch(recog_case, arrival, group):
    """streaming pushes with the band matcher (r = 16, the whole-row kernel with a device-side batch size; r = 10 the
    thread form): every segment-0 event equals batch recognition with the same matcher, and every event equals the
    oracle's get_mfcc of its segment, then its banded dtw and argmin"""
    ora = ob.best_oracle()
    S, L, T = 24, 40000, 20
    bank = recog_case["bank20"]
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDD000, 3)
    pcm[3] = 2048                                            # a silent stream: no event
    for r in (16, 10):
        hs = [handle(bank, T, BAND, r) for _ in range(2 if group else 1)]
        pool = sr_b200.StreamPool(hs if group else hs[0], S, L, 2400)
        events = _stream_events(pool, pcm, arrival, np.random.default_rng(0xE5 + r))
        seg, atap = pool.segments()
        pool.close()
        closed = [(s, k) for s in range(S) for k in range(3) if seg[s, k, 1] != ob.NULL]
        assert sorted((e["stream"], e["segment"]) for e in events) == closed and len(closed) >= 2 * S
        batch = hs[0].recognise(pcm, 2400)
        assert np.array_equal(batch["seg_off"][:, 0], seg[:, 0])
        for e in events:
            s, k = e["stream"], e["segment"]
            if k == 0:
                got = tuple(e[q] for q in ("best_idx", "best_dis", "cmd", "status"))
                assert got == tuple(int(batch[q][s]) for q in ("best_idx", "best_dis", "cmd", "status")), (r, e)
            f = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
            assert e["frm_num"] == int(f["frm_num"][0]), (r, e)
            if e["frm_num"] == 0:
                assert (e["status"], e["best_idx"], e["best_dis"]) == (2, 0, ob.NULL), (r, e)
                continue
            sc, _ = ob.port().dtw_batch(f, bank, T, 4096, check_sign=1, band_r=r)
            i = int(np.argmin(sc[0]))
            assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == (0, i, int(sc[0, i]), i // 4), (r, e)
        for h in hs:
            h.close()


# ---- handles that disagree ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_multi_and_group_calls_refuse_handles_with_different_matchers(recog_case):
    """sr_recognise_batch_multi and sr_stream_group_push* fail when their handles differ in the matcher (greedy vs band,
    or two radii), and run once the matchers agree"""
    bank = recog_case["bank20"]
    pcm = recog_case["pcm"][:64]
    for second in ((0, 0), (sr_b200.DTW_BAND, 15)):
        a, b = handle(bank, 20, BAND, 16), handle(bank, 20)
        b.set_match(*second)
        with pytest.raises(sr_b200.SrError):
            sr_b200.recognise_multi([a, b], pcm, 2400)
        pool = sr_b200.StreamPool([a, b], 8, 8000, 2400)
        with pytest.raises(sr_b200.SrError):
            pool.push(np.ascontiguousarray(pcm[:8, :800]))
        with pytest.raises(sr_b200.SrError):
            pool.push_ragged(np.ascontiguousarray(pcm[:8, :800]), np.full(8, 800, np.uint32))
        b.set_match(sr_b200.DTW_BAND, 16)
        pool.push(np.ascontiguousarray(pcm[:8, :800]))
        pool.close()
        out = sr_b200.recognise_multi([a, b], pcm, 2400)
        assert np.array_equal(out["score"], a.recognise(pcm, 2400)["score"])
        a.close()
        b.close()
