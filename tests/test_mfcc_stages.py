"""get_mfcc stage by stage (K1 mfcc_kernel_s16, K5 mfcc_geomb_kernel and the shared MFCC core). The final
coefficients hide most of the frame's arithmetic: log*100 is coarse (thresholds about 1 % apart), so a filter sum that
is off by a few units changes the output only when it sits within those units of a threshold, and the usual inputs
(speech, random PCM, board captures) keep every filter sum above 10 000. This file

  * pins the plain stage reference of tests/mfcc_ref.py to the oracle (and to the reference's own build where it
    exists) on the usual inputs and on the frames below, in both geometries;
  * builds one-frame inputs on which moving any one filter sum by +1 or by -1 changes the coefficients, asserting on the
    CPU that they reach that regime, and runs them through every MFCC entry point on the GPU;
  * checks the kernels' float estimates of exact integer steps, log100 and the magnitude, over their whole domains."""
import ctypes as C
import os

import numpy as np
import pytest

import mfcc_ref as mr
import oracle_bind as ob
import sr_b200

HERE = os.path.dirname(os.path.abspath(__file__))
CAPS = np.load(os.path.join(HERE, "golden", "captures.npz"))
GEOMS = {"A": mr.GEOM_A, "B": mr.GEOM_B}


def _port_mfcc(g):
    po = ob.port()
    return po.mfcc_batch if g.name == "A" else po.mfcc_geom_b_batch


def _one_frame_batch(g):
    """the exposing frames as one-frame segments [1, 1 + frame) of rows [x[-1], samples...]"""
    rows, mid, st = mr.exposing_frames(g)
    seg = np.tile(np.array([1, g.frame + 1], np.uint32), (len(rows), 1))
    atap = np.zeros(len(rows), ob.ATAP_DTYPE)
    atap["mid_val"] = mid
    return np.ascontiguousarray(rows), seg, atap, st


def _usual_inputs(g):
    """the board captures cut into segments of at most 119 frames, random 12-bit PCM with a random mid_val, and
    full-range u16 PCM: (pcm, seg, atap)"""
    rng = np.random.default_rng(0x57A6)
    span = g.frame + 118 * g.hop
    rows, segs, mids = [], [], []
    for name in CAPS.files:
        x = CAPS[name]
        mid = int(round(float(x[:2400].mean())))
        for st in range(1, len(x) - g.frame, span):
            rows.append(x)
            segs.append((st, min(st + span, len(x))))
            mids.append(mid)
    U = max(len(r) for r in rows)
    pcm = np.zeros((len(rows) + 8, U), np.uint16)
    for i, r in enumerate(rows):
        pcm[i, :len(r)] = r
    pcm[len(rows):len(rows) + 4] = rng.integers(0, 4096, (4, U))
    pcm[len(rows) + 4:] = rng.integers(0, 65536, (4, U))
    for _ in range(8):
        st = int(rng.integers(1, 2000))
        segs.append((st, st + int(rng.integers(g.frame, span))))
    mids += rng.integers(0, 4096, 4).tolist() + rng.integers(0, 65536, 4).tolist()
    atap = np.zeros(len(pcm), ob.ATAP_DTYPE)
    atap["mid_val"] = mids
    return pcm, np.array(segs, np.uint32), atap


# ---- CPU: the stage reference against the oracle, and the reach of the exposing frames ------------------------------
@pytest.mark.parametrize("geom", ["A", "B"])
def test_stage_reference_equals_oracle(geom):
    """the stage reference's coefficients equal the oracle's get_mfcc bit for bit on the board captures, random and
    full-range PCM and the exposing frames; in the reference geometry also the reference's own get_mfcc where it is
    built, except on frames with a filter sum of 0, where the reference takes log(0) (DESIGN §3)"""
    g = GEOMS[geom]
    cases = [_usual_inputs(g), _one_frame_batch(g)[:3]]
    for pcm, seg, atap in cases:
        ftr, sums, rows = mr.mfcc_batch(pcm, seg, atap, g)
        assert (ftr["frm_num"] > 0).all()
        assert ob.ftr_equal(ftr, _port_mfcc(g)(pcm, seg, atap))
        if geom == "A" and ob.have_ref():
            zero = np.zeros(len(pcm), bool)
            zero[rows[(sums == 0).any(axis=1)]] = True
            keep = ~zero
            assert keep.sum() >= len(pcm) // 5
            assert ob.ftr_equal(ftr[keep], ob.ref().mfcc_batch(pcm[keep], seg[keep], atap[keep]))


def test_usual_inputs_keep_filter_sums_large():
    """why the exposing frames exist: on the usual inputs no filter sum is below 100, and few sums sit where +-1
    changes a coefficient"""
    for g in GEOMS.values():
        pcm, seg, atap = _usual_inputs(g)
        _, sums, _ = mr.mfcc_batch(pcm, seg, atap, g)
        s = sums.astype(np.int64)
        assert not ((s >= 1) & (s <= 99)).any(), g.name


@pytest.mark.parametrize("geom", ["A", "B"])
def test_exposing_frames_reach_the_sensitive_regime(geom):
    """every (filter, sign) is exposed by at least 4 frames; sums sit exactly on thresholds thr[L] and one below them;
    sums of 0 mix with nonzero ones; all-zero frames at mid_val 0, 2 048 and 65 535; zero-magnitude bins beside
    nonzero ones (the pw = 0 path of mag10_small); in the reference geometry sums of 1 .. 99 in most filters"""
    g = GEOMS[geom]
    rows, seg, atap, st = _one_frame_batch(g)
    s = st["sums"].astype(np.int64)
    ex = mr.exposure(st["sums"], g)
    assert ex.sum(axis=0).min() >= 4, ex.sum(axis=0)
    thr = mr.THR[100:].astype(np.int64)
    assert np.isin(s, thr).sum() >= 4 and np.isin(s, thr - 1).sum() >= 4
    assert ((s == 0).any(axis=1) & (s > 0).any(axis=1)).sum() >= 4
    zero = (s == 0).all(axis=1)
    assert set(atap["mid_val"][zero].tolist()) >= {0, 2048, 65535}
    assert (st["win"][zero] == 0).all()
    assert ((st["mag"] == 0).any(axis=1) & (st["mag"] > 0).any(axis=1)).sum() >= 20
    assert set(atap["mid_val"].tolist()) >= {0, 2048, 65535}
    if geom == "A":
        small = (s >= 1) & (s <= 99)
        assert (small.any(axis=0)).sum() >= 16 and small.any(axis=1).sum() >= 50
        assert ex[small.any(axis=1)].any(axis=(1, 2)).all()


# ---- GPU: the exposing frames through every MFCC entry point, and the whole-domain checks ---------------------------
def _to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to("cuda:0")


@pytest.mark.gpu
def test_exposing_frames_on_every_mfcc_call(handle):
    """K1 through sr_mfcc_batch, sr_mfcc_batch_dev, the drop-in get_mfcc and sr_mfcc_long_batch, bit for bit with the
    oracle, on frames where a one-unit error in any filter sum changes the coefficients"""
    import torch
    pcm, seg, atap, st = _one_frame_batch(mr.GEOM_A)
    want = ob.port().mfcc_batch(pcm, seg, atap)
    assert (want["frm_num"] == 1).all()
    assert np.array_equal(want["mfcc_dat"][:, :12], st["mfcc"])
    assert ob.ftr_equal(handle.mfcc(pcm, seg, atap), want)
    ft = torch.full((len(pcm) * sr_b200.FTR_BYTES,), 0x5A, dtype=torch.uint8, device="cuda:0")
    pd, sd, ad = _to_dev(pcm), _to_dev(seg), _to_dev(atap)
    handle.mfcc_dev(pd.data_ptr(), pcm.shape[1], len(pcm), sd.data_ptr(), 2, ad.data_ptr(), ft.data_ptr())
    torch.cuda.synchronize()
    assert ob.ftr_equal(ft.cpu().numpy().view(sr_b200.FTR_DTYPE), want)
    feat, frm = handle.mfcc_long(pcm, seg, atap)
    assert (frm == 1).all() and np.array_equal(feat[:, 0, :], st["mfcc"])
    L = sr_b200.lib()
    f = np.zeros(len(pcm), sr_b200.FTR_DTYPE)
    for b in range(len(pcm)):                          # valid->start = sample 1 (x[-1] = sample 0), valid->end = row end
        vv = sr_b200.ValidTag(pcm[b].ctypes.data + 2, pcm[b].ctypes.data + 2 * pcm.shape[1])
        L.get_mfcc(C.byref(vv), f[b:b + 1].ctypes.data_as(C.c_void_p), atap[b:b + 1].ctypes.data_as(C.c_void_p))
    assert ob.ftr_equal(f, want)


@pytest.mark.gpu
def test_exposing_frames_geom_b():
    """K5 (mfcc_geomb_kernel) through sr_mfcc_batch and sr_mfcc_batch_dev on its own exposing frames"""
    import torch
    pcm, seg, atap, st = _one_frame_batch(mr.GEOM_B)
    want = ob.port().mfcc_geom_b_batch(pcm, seg, atap)
    assert (want["frm_num"] == 1).all() and np.array_equal(want["mfcc_dat"][:, :12], st["mfcc"])
    h = sr_b200.Handle(0)
    h.set_geometry(1)
    assert ob.ftr_equal(h.mfcc(pcm, seg, atap), want)
    ft = torch.full((len(pcm) * sr_b200.FTR_BYTES,), 0x5A, dtype=torch.uint8, device="cuda:0")
    pd, sd, ad = _to_dev(pcm), _to_dev(seg), _to_dev(atap)
    h.mfcc_dev(pd.data_ptr(), pcm.shape[1], len(pcm), sd.data_ptr(), 2, ad.data_ptr(), ft.data_ptr())
    torch.cuda.synchronize()
    assert ob.ftr_equal(ft.cpu().numpy().view(sr_b200.FTR_DTYPE), want)
    h.close()


@pytest.mark.gpu
def test_log100_whole_domain(handle):
    """the kernels' log100 (float estimate, then a downward and an upward correction loop) equals a binary search over
    the same threshold table for every u32 v, log(0) pinned to 0 included"""
    bad = C.c_uint64(123)
    assert sr_b200.lib().sr_debug_log100_mismatches(handle._h, 0, 1 << 32, C.byref(bad)) == 0
    assert bad.value == 0


@pytest.mark.gpu
def test_magnitude_whole_domain(handle):
    """mag10_small over every (re, im) with |re|, |im| <= 8 209 (every bin the pruned FFT of K1 can produce), and mag10
    over every s16 pair (the generic FFT and K5), equal (u32)(sqrtf((float)pw) * 10) with IEEE steps: 0 for pw = 0 and
    for the one negative s32 pw, re = im = -32768"""
    L = sr_b200.lib()
    for which, n in ((0, 16419 ** 2), (1, 1 << 32)):
        bad = C.c_uint64(123)
        assert L.sr_debug_mag10_mismatches(handle._h, which, 0, n, C.byref(bad)) == 0
        assert bad.value == 0, which
