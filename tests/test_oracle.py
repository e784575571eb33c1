"""The oracle restatement (oracle/sr_oracle.c) pinned against (a) the golden vectors produced by executing
the reference's own C (tests/golden/golden.npz, made by tests/golden/make_golden.py) and (b) when the
prebuilt oracle/_ref/libref.so is present, the reference itself on random / synthetic inputs. CPU only."""
import os

import numpy as np
import pytest

import oracle_bind as ob
import sr_b200

HERE = os.path.dirname(os.path.abspath(__file__))
CAPS = np.load(os.path.join(HERE, "golden", "captures.npz"))
GOLD = np.load(os.path.join(HERE, "golden", "golden.npz"))


def _need_ref():
    """evaluated at run time (after the session build fixture), not at collection time"""
    if not ob.have_ref():
        pytest.skip("oracle/_ref/libref.so not built (reference tree not mounted and no prebuilt .so)")



@pytest.mark.parametrize("name", ["stm32_123", "stm32_456", "stm32_noise", "stm32_voice_123", "v1"])
def test_port_matches_golden_on_board_captures(name):
    o = ob.port()
    pcm = CAPS[name]
    atap = o.noise_atap(pcm, 2400)
    assert atap.tobytes() == GOLD[name + "/atap"].tobytes()
    seg = o.vad(pcm, len(pcm), atap)
    assert seg.tolist() == GOLD[name + "/seg"].tolist()
    ftrs = []
    for k in range(3):
        key = "%s/ftr%d" % (name, k)
        if key in GOLD:
            f = o.mfcc_batch(pcm.reshape(1, -1), seg[2 * k:2 * k + 2].reshape(1, 2), atap)
            assert ob.ftr_equal(f, GOLD[key])
            ftrs.append(f)
    if name + "/dtw" in GOLD:
        bank = np.concatenate(ftrs).view(np.uint8).reshape(len(ftrs), -1)
        sc, _ = o.dtw_batch(np.concatenate(ftrs), bank, len(ftrs), 2860)
        assert sc.tolist() == GOLD[name + "/dtw"].tolist()


def test_port_matches_golden_on_synthetic_batch():
    o = ob.port()
    pcm = sr_b200.synth_pcm_host(24, 8000, 0x5EED0000)
    tpl = sr_b200.synth_pcm_host(8, 8000, 0x7E3A0000)
    assert [int(pcm.astype(np.uint64).sum()), int(tpl.astype(np.uint64).sum())] == GOLD["synth/pcm_sum"].tolist()
    bank = GOLD["synth/bank"]
    out = o.recognise_batch(pcm, 2400, bank, 8, 4096, nthreads=4)
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
        assert np.array_equal(out[k], GOLD["synth/" + k]), k
    assert ob.ftr_equal(out["ftr"], GOLD["synth/ftr"])
    pcm5 = sr_b200.synth_pcm_host(4, 40000, 0x5EED5000, 3)
    out5 = o.recognise_batch(pcm5, 2400, bank, 8, 4096)
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
        assert np.array_equal(out5[k], GOLD["synth5/" + k]), k
    assert (out5["seg_off"].reshape(4, 6) != ob.NULL).all()        # exactly max_vc_con words found


def test_port_fft_equals_reference_build_on_random_inputs():
    _need_ref()
    rng = np.random.default_rng(11)
    x = rng.integers(0, 2 ** 32, (64, 1024), dtype=np.uint32)           # arbitrary complex s16 pairs
    x[:8] = 0
    x[8:16, :160] = rng.integers(-32768, 32768, (8, 160)).astype(np.int16).astype(np.uint16)
    assert np.array_equal(ob.port().fft_raw(x), ob.ref().fft_raw(x))
    fr = rng.integers(-32768, 32768, (32, 160)).astype(np.int16)
    assert np.array_equal(ob.port().fft_mag(fr), ob.ref().fft_mag(fr))


def test_port_equals_reference_build_on_noisy_and_extreme_pcm():
    _need_ref()
    rng = np.random.default_rng(5)
    B, U = 12, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0xABCD0000)
    pcm[0] = rng.integers(0, 4096, U)                 # white noise, full scale
    pcm[1] = rng.integers(0, 65536, U)                # beyond 12 bit: exercises the s16 / u32 wraps
    pcm[2, :] = 2048                                  # dead silent: n_thl = 0
    pcm[3, 2400:] = np.where(np.arange(U - 2400) % 2 == 0, 0, 4095)    # maximal zero-crossing rate
    pcm[4, 3000:7900] = rng.integers(0, 4096, 4900)  # speech runs into the end: segment never closes
    tpl = sr_b200.synth_pcm_host(6, U, 0x7E3A0000)
    r, p = ob.ref(), ob.port()
    e = r.recognise_batch(tpl, 2400, None, 0, 4096)
    bank = sr_b200.make_bank(e["ftr"], valid=[1, 1, 0, 1, 1, 1])
    a, b = r.recognise_batch(pcm, 2400, bank, 6, 4096), p.recognise_batch(pcm, 2400, bank, 6, 4096, nthreads=3)
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
        assert np.array_equal(a[k], b[k]), k
    assert ob.ftr_equal(a["ftr"], b["ftr"])
    # fixed-segment MFCC on the extreme rows (VAD bypassed)
    seg = np.tile(np.array([80, 8000], np.uint32), (B, 1))
    atap = np.zeros(B, ob.ATAP_DTYPE)
    atap["mid_val"] = 2048
    assert ob.ftr_equal(r.mfcc_batch(pcm, seg, atap), p.mfcc_batch(pcm, seg, atap, nthreads=2))


def test_port_dtw_equals_reference_build_on_random_features():
    _need_ref()
    raw = sr_b200.synth_ftr_host(40, 0xD7A00000, 1, 119)
    ftr = raw.view(ob.FTR_DTYPE).reshape(-1)
    bank = sr_b200.synth_ftr_host(23, 0xD7A10000, 1, 119, stride=4096)
    a, _ = ob.ref().dtw_batch(ftr, bank, 23, 4096)
    b, cells = ob.port().dtw_batch(ftr, bank, 23, 4096, nthreads=2)
    assert np.array_equal(a, b) and cells > 0
    assert (a == ob.NULL).any() and (a != ob.NULL).any()          # the 2:1 guard fires on some pairs


def test_port_get_mdl_equals_reference_build():
    _need_ref()
    f1 = sr_b200.synth_ftr_host(40, 0xAA00, 1, 59).view(ob.FTR_DTYPE).reshape(-1)        # paths <= 117 points: the
    f2 = sr_b200.synth_ftr_host(40, 0xBB00, 1, 59).view(ob.FTR_DTYPE).reshape(-1)        # reference does not bound its writes
    m1, d1 = ob.ref().get_mdl(f1, f2)
    m2, d2 = ob.port().get_mdl(f1, f2)
    assert np.array_equal(d1, d2) and ob.ftr_equal(m1, m2) and (d1 != ob.NULL).any() and (d1 == ob.NULL).any()


@pytest.mark.parametrize("which", ["port", "ref"])
def test_sample0_inputs_reach_the_case_and_recognise_pinned_is_recognise_batch(which):
    """plant_sample0 and recognise_pinned are the inputs and the reference of the GPU tests of x[-1] at sample 0
    (test_gpu_parity.py, *sample0*). Identity: on utterances none of whose segments starts at sample 0, recognise_pinned
    equals the oracle's own recognise_batch in every field. Reach: VAD opens segment 0 of every planted utterance at
    sample 0, with 1..119 frames, and no other. Sensitivity: every planted utterance's features differ between x[-1] =
    mid_val, 0 and the preceding row's last sample, so a kernel that read either would fail those tests."""
    if which == "ref":
        _need_ref()
    o = ob.port() if which == "port" else ob.ref()
    B, U, T = 48, 8000, 10
    tpl = sr_b200.synth_pcm_host(T, U, 0x5A0B0000)
    ob.plant_sample0(tpl, [1, 4, 7], 3)
    e = ob.recognise_pinned(o, tpl, 2400, None, 0, 4096)
    assert (e["status"] == 0).all()
    bank = sr_b200.make_bank(e["ftr"])
    pcm = sr_b200.synth_pcm_host(B, U, 0x5A0A0000)
    pcm[5] = 2048                                      # VAD fails: status 1
    want = o.recognise_batch(pcm, 2400, bank, T, 4096)
    got = ob.recognise_pinned(o, pcm, 2400, bank, T, 4096)
    assert (want["seg_off"][:, :, 0] != 0).all() and set(want["status"].tolist()) == {0, 1}
    for k in want:
        if k == "ftr":
            assert ob.ftr_equal(got[k], want[k])
        else:
            assert np.array_equal(got[k], want[k]), k
    rows = [0, 1, 2, 9, 10, 23, 24, 46, 47]
    ob.plant_sample0(pcm, rows, 4)
    p = ob.recognise_pinned(o, pcm, 2400, bank, T, 4096)
    planted = np.isin(np.arange(B), rows)
    assert ((p["seg_off"][:, 0, 0] == 0) == planted).all()
    assert (p["status"][rows] == 0).all() and (p["ftr"]["frm_num"][rows] >= 1).all() and (p["ftr"]["frm_num"][rows] <= 119).all()
    assert (p["best_dis"][rows] != ob.NULL).any()      # the planted templates are in reach of the 2:1 guard (DTW.C:133)
    seg = p["seg_off"][rows, 0, :] + 1
    base = ob.pinned_rows(pcm[rows], p["atap"][rows])
    feats = {}
    for name, x1 in (("mid", None), ("zero", 0), ("before", "prev")):
        r1 = base.copy()
        if x1 == "prev":
            r1[:, 0] = [pcm[r - 1, -1] if r else 4095 for r in rows]
        elif x1 is not None:
            r1[:, 0] = x1
        feats[name] = o.mfcc_batch(r1, seg, p["atap"][rows])
    assert ob.ftr_equal(feats["mid"], p["ftr"][rows])
    for i, r in enumerate(rows):
        assert r == 0 or pcm[r - 1, -1] == 4095
        for a, b in (("mid", "zero"), ("mid", "before"), ("zero", "before")):
            assert not ob.ftr_equal(feats[a][i:i + 1], feats[b][i:i + 1]), (r, a, b)


def test_dtw_band_oracle_properties():
    """dtw_band is our own extension (parity unpinned by the reference): sanity properties only"""
    raw = sr_b200.synth_ftr_host(6, 0xD7A20000, 50, 100)
    ftr = raw.view(ob.FTR_DTYPE).reshape(-1)
    o = ob.port()
    sc, cells = o.dtw_batch(ftr, raw, 6, 2860, band_r=10)
    assert (np.diag(sc) == 0).all() and cells > 0
    wide, _ = o.dtw_batch(ftr, raw, 6, 2860, band_r=200)
    ok = (sc != ob.NULL) & (wide != ob.NULL)
    assert (wide[ok] <= sc[ok]).all()                               # a wider band can only lower the DP optimum


def test_generic_radix4_fft_reproduces_the_1024_point_restatement():
    """oracle/cr4_fft_generic.c (the asm's algorithm for N = 64 / 256 / 1024) at N = 1024 == the register-level
    restatement of cr4_fft_1024_stm32.s -- and, where the reference is compiled, == libref's FFT: this pins the
    generalisation whose N = 256 instance carries the GEOM_B extension"""
    import oracle_bind as ob
    rng = np.random.default_rng(256)
    x = rng.integers(0, 2 ** 32, (24, 1024), dtype=np.uint64).astype(np.uint32)
    x[0] = 0x80008000
    x[1] = 0x7FFF7FFF
    x[2, :160] = rng.integers(0, 65536, 160).astype(np.uint32)
    x[2, 160:] = 0
    po = ob.port()
    want = po.fft_raw(x)
    assert np.array_equal(po.fft_raw_n(x, 1024), want)
    if ob.have_ref():
        assert np.array_equal(ob.ref().fft_raw(x), want)
    # smaller sizes: DC and single-tone sanity (|error| vs the exact DFT/N stays within a few LSB like the 1024-point routine)
    for N in (64, 256):
        n = np.arange(N)
        tone = np.round(8000 * np.cos(2 * np.pi * 5 * n / N)).astype(np.int64)
        packed = (tone & 0xFFFF).astype(np.uint32).reshape(1, N)
        out = po.fft_raw_n(packed, N)[0]
        re = (out & 0xFFFF).astype(np.int16).astype(np.int64)
        im = (out >> 16).astype(np.int16).astype(np.int64)
        exact = np.fft.fft(tone) / N
        assert np.abs(re - exact.real).max() <= 8 and np.abs(im - exact.imag).max() <= 8
        assert abs(re[5] - 4000) <= 8 and abs(re[N - 5] - 4000) <= 8


def test_bitmap_endpoint_fsm_equals_sequential_fsm_on_every_prefix():
    """The endpoint FSM of VAD.C:164-216 as the kernels evaluate it on one window from a fresh state
    (sr_vad_core.cuh::long_fsm_window's a8 / z11 bitmaps and find_first, as K0 runs it through vad_window: 8 consecutive
    active frames open a segment at the first of them, 11 consecutive inactive frames close it at the first of those,
    the first 3 segments kept) against the sequential state machine -- on random activity patterns and on EVERY prefix of
    them: a window that ends at any frame yields exactly the decisions the sequential FSM has taken by then, which is
    what lets the streaming kernels carry the FSM's state from push to push."""
    rng = np.random.default_rng(164)

    def sequential(act):
        seg = [None] * 6
        cur = front = back = con = 0
        for k, a in enumerate(act):
            i = 80 * k
            if a:                                               # VAD.C:164-187
                if cur == 0:
                    cur, front = 1, 1
                elif cur == 1:
                    front += 1
                    if front >= 8:
                        cur, seg[2 * con], front = 2, i - 7 * 80, 0
                elif cur == 3:
                    back, cur = 0, 2
            else:                                               # VAD.C:188-216
                if cur == 2:
                    cur, back = 3, 1
                elif cur == 3:
                    back += 1
                    if back >= 11:
                        cur, back = 0, 0
                        seg[2 * con + 1] = i - 11 * 80 + 160
                        con += 1
                        if con == 3:
                            break
                elif cur == 1:
                    front, cur = 0, 0
        return seg

    def bitmap(act):
        n = len(act)
        aw = sum(1 << k for k, a in enumerate(act) if a)
        vmask = (1 << n) - 1
        a8 = aw
        for s in (1, 2, 4):
            a8 &= a8 >> s
        z = ~aw & vmask
        z8 = z
        for s in (1, 2, 4):
            z8 &= z8 >> s
        z11 = z8 & (z8 >> 3)
        seg, cur = [None] * 6, 0

        def first(bits, frm):
            bits >>= frm
            return -1 if bits == 0 else frm + (bits & -bits).bit_length() - 1
        for sgi in range(3):
            p = first(a8, cur)
            if p < 0:
                break
            seg[2 * sgi] = 80 * p
            q = first(z11, p + 8)
            if q < 0:
                break
            seg[2 * sgi + 1] = 80 * q + 80
            cur = q + 11
        return seg

    for trial in range(60):
        n = int(rng.integers(1, 500))
        p_on = float(rng.choice([0.1, 0.5, 0.8, 0.95]))
        act, state = [], 0
        for _ in range(n):                                       # bursty activity: runs of speech and silence
            if rng.random() < 0.08:
                state ^= 1
            act.append(bool(state) if rng.random() < p_on else bool(rng.integers(0, 2)))
        for m in list(range(0, n + 1, 7)) + [n]:
            assert bitmap(act[:m]) == sequential(act[:m]), (trial, m)
