"""The per-call rules of the C-ABI's host-buffer and device-pointer entry points: how many kernels one call launches and
which of them it times, which arguments are checked before the zero-size early return, and that a workspace grown or
reused by an earlier call of another size never changes a result."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as ob
import sr_b200

pytestmark = pytest.mark.gpu

U, T = 8000, 6
VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL, DTW_BAND = range(7)


def _handle(bank=True):
    h = sr_b200.Handle(0)
    h.timing_enable(512)
    h.set_transport(0)
    if bank:
        b, st = h.enrol(sr_b200.synth_pcm_host(T, U, 0x7E3A0000), 2400)
        assert (st == 0).all()
        h.set_bank(b, T, 4096)
    h.timing_collect()
    return h


@pytest.fixture(scope="module")
def h():
    h = _handle()
    yield h
    h.close()


@pytest.fixture(scope="module")
def data():
    B = 12
    pcm = sr_b200.synth_pcm_host(B, U, 0x40C0)
    hh = _handle(bank=False)
    atap = hh.noise_atap(pcm, 2400)
    seg = hh.vad(pcm, atap)
    ftr = hh.mfcc(pcm, seg, atap)
    hh.close()
    assert (ftr["frm_num"] > 0).any()
    return {"pcm": pcm, "atap": atap, "seg": seg, "ftr": ftr}


def _account(h, fn):
    """(launches, timing tags) of fn(); the handle's timing records are drained before and after"""
    h.timing_collect()
    l0 = h.launch_count()
    fn()
    tags = [t for t, _ in h.timing_collect()]
    return h.launch_count() - l0, tags


def _rc(h, fn, *args):
    """return code of a raw C-ABI call on h, and the handle's error text"""
    return getattr(sr_b200.lib(), fn)(h._h, *args), sr_b200.lib().sr_last_error(h._h)


def _dev(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to("cuda:0")
    torch.cuda.synchronize()
    return t


def _zeros_dev(nbytes):
    import torch
    t = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    return t


# ---- launches and timing records of one call ------------------------------------------------------------------------
def test_host_buffer_call_accounting(h, data):
    pcm, atap, seg, ftr = data["pcm"], data["atap"], data["seg"], data["ftr"]
    B = pcm.shape[0]
    assert _account(h, lambda: h.noise_atap(pcm, 2400)) == (1, [VAD_])
    assert _account(h, lambda: h.vad(pcm, atap)) == (1, [VAD_])
    assert _account(h, lambda: h.mfcc(pcm, seg, atap)) == (1, [MFCC_])
    assert _account(h, lambda: h.dtw(ftr)) == (3, [BEST_INIT, DTW, BEST_FINAL])
    assert _account(h, lambda: h.dtw(ftr, sr_b200.DTW_BAND, 8)) == (3, [BEST_INIT, DTW_BAND, BEST_FINAL])
    assert _account(h, lambda: h.dtw(ftr, want_best=False)) == (1, [DTW])
    assert _account(h, lambda: h.recognise(pcm, 2400)) == (6, [VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL])
    assert _account(h, lambda: h.recognise(pcm, 2400, want=("ftr", "status"))) == (4, [VAD_, MFCC_, STATUS, DTW])
    assert _account(h, lambda: h.enrol(pcm, 2400)) == (4, [VAD_, MFCC_, STATUS])
    f2 = np.ascontiguousarray(ftr[::-1])
    assert _account(h, lambda: h.get_mdl(ftr, f2)) == (1, [])
    assert _account(h, lambda: h.fft_mag(np.ones((B, 160), np.int16))) == (1, [])
    assert _account(h, lambda: h.fft_raw(np.ones((B, 1024), np.uint32))) == (1, [])
    assert _account(h, lambda: h.fft_raw_n(np.ones((B, 256), np.uint32), 256)) == (1, [])
    rows = ftr["mfcc_dat"][:, :12].copy()
    assert _account(h, lambda: h.get_dis(rows, rows[::-1].copy())) == (1, [])
    v = np.arange(B, dtype=np.uint16)
    out = np.zeros(B, np.uint8)
    assert _account(h, lambda: _rc(h, "sr_dtw_limit_batch", *[x.ctypes.data for x in (v, v, v + 5, v + 9)], B,
                                   out.ctypes.data)) == (1, [])
    packed = np.arange(3 * 64, dtype=np.uint8)
    assert _account(h, lambda: h.unpack12(packed, 128)) == (1, [])
    bad = C.c_uint64(7)
    n, tags = _account(h, lambda: _rc(h, "sr_debug_sqrt_mismatches", 0x3F800000, 0x3F810000, C.byref(bad)))
    assert tags == [] and bad.value == 0
    bad = C.c_uint64(7)
    n, tags = _account(h, lambda: _rc(h, "sr_debug_log100_mismatches", 0, 1 << 16, C.byref(bad)))
    assert tags == [] and bad.value == 0
    for which in (0, 1):
        bad = C.c_uint64(7)
        n, tags = _account(h, lambda: _rc(h, "sr_debug_mag10_mismatches", which, 0, 1 << 16, C.byref(bad)))
        assert tags == [] and bad.value == 0


def test_dtw_without_templates_launches_only_the_argmin(data):
    h = _handle(bank=False)
    assert _account(h, lambda: h.dtw(data["ftr"])) == (2, [BEST_INIT, BEST_FINAL])
    assert _account(h, lambda: h.dtw(data["ftr"], want_best=False)) == (0, [])
    h.close()


def test_recognise_chunks_and_packed_transport(h):
    """one launch sequence per chunk, and one untimed expansion launch per chunk that crossed PCIe packed"""
    B = 3 * 2096 + 8                                   # four chunks of 8 000-sample utterances (fewer are never packed)
    pcm = sr_b200.synth_pcm_host(B, U, 0x2C2C)
    per_chunk = [VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL]
    for mode in (0, 1):
        h.set_transport(mode)
        n, tags = _account(h, lambda: h.recognise(pcm, 2400))
        packed, plain, _ = h.transport_stats()
        assert packed + plain == 4 and (mode == 1 or packed == 0)
        assert (n, tags) == (24 + packed, per_chunk * 4)
    h.set_transport(0)


def test_device_pointer_call_accounting(h, data):
    pcm, atap, seg, ftr = data["pcm"], data["atap"], data["seg"], data["ftr"]
    B = pcm.shape[0]
    pcm_d, atap_d, seg_d, ftr_d = _dev(pcm), _dev(atap), _dev(seg), _dev(ftr)
    at, sg, ft = _zeros_dev(B * 12), _zeros_dev(B * 24), _zeros_dev(B * 2860)
    score, bi, bd = _zeros_dev(B * T * 4), _zeros_dev(B * 4), _zeros_dev(B * 4)
    assert _account(h, lambda: h.noise_atap_dev(pcm_d.data_ptr(), U, B, 2400, at.data_ptr())) == (1, [VAD_])
    assert _account(h, lambda: h.vad_dev(pcm_d.data_ptr(), U, B, U, atap_d.data_ptr(), sg.data_ptr())) == (1, [VAD_])
    assert _account(h, lambda: h.mfcc_dev(pcm_d.data_ptr(), U, B, seg_d.data_ptr(), 6, atap_d.data_ptr(),
                                          ft.data_ptr())) == (1, [MFCC_])
    assert _account(h, lambda: h.dtw_dev(ftr_d.data_ptr(), B, 0, 0, score.data_ptr(), bi.data_ptr(),
                                         bd.data_ptr())) == (3, [BEST_INIT, DTW, BEST_FINAL])
    assert _account(h, lambda: h.dtw_dev(ftr_d.data_ptr(), B, sr_b200.DTW_BAND, 8, score.data_ptr(), None,
                                         bd.data_ptr())) == (3, [BEST_INIT, DTW_BAND, BEST_FINAL])
    assert _account(h, lambda: h.dtw_dev(ftr_d.data_ptr(), B, 0, 0, score.data_ptr(), None, None)) == (1, [DTW])
    o = {"atap": at, "seg_off": sg, "ftr": ft, "score": score, "best_idx": bi, "best_dis": bd,
         "cmd": _zeros_dev(B * 4), "status": _zeros_dev(B)}
    assert _account(h, lambda: h.recognise_dev(pcm_d.data_ptr(), U, B, 2400, **{k: v.data_ptr() for k, v in o.items()})) \
        == (6, [VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL])
    assert _account(h, lambda: h.recognise_dev(pcm_d.data_ptr(), U, B, 2400, ftr=ft.data_ptr())) \
        == (4, [VAD_, MFCC_, STATUS, DTW])
    h.sync()
    assert np.array_equal(sg.cpu().numpy().view(np.uint32).reshape(seg.shape), h.vad(pcm, atap))   # recognise_dev's segments


# ---- argument errors and the zero-size early return -----------------------------------------------------------------
def test_null_pointer_with_work_fails(h):
    p = np.zeros(1 << 16, np.uint8)
    a = p.ctypes.data
    cases = [("sr_noise_atap_batch", (None, U, 1, 2400, a)), ("sr_noise_atap_batch", (a, U, 1, 2400, None)),
             ("sr_vad_batch", (a, U, 1, U, None, a)), ("sr_vad_batch", (a, U, 1, U, a, None)),
             ("sr_mfcc_batch", (a, U, 1, a, 2, a, None)), ("sr_mfcc_batch", (a, U, 1, None, 2, a, a)),
             ("sr_dtw_batch", (None, 1, 0, 0, a, a, a)),
             ("sr_recognise_batch", (None, U, 1, 2400, C.byref(sr_b200.RecogOut()))),
             ("sr_recognise_batch", (a, U, 1, 2400, None)),
             ("sr_enrol_batch", (a, U, 1, 2400, None, 4096, a)), ("sr_enrol_batch", (None, U, 1, 2400, a, 4096, a)),
             ("sr_get_mdl_batch", (a, None, 1, a, a)), ("sr_get_mdl_batch", (a, a, 1, None, a)),
             ("sr_fft_mag_batch", (None, 160, 1, a)), ("sr_fft_mag_batch", (a, 160, 1, None)),
             ("sr_fft_raw_batch", (a, 1, None)), ("sr_get_dis_batch", (a, None, 1, a)),
             ("sr_debug_fft_raw_n", (None, 256, 1, a)), ("sr_debug_fft_raw_n", (a, 1024, 1, None)),
             ("sr_dtw_limit_batch", (a, a, None, a, 1, a)), ("sr_debug_unpack12", (a, 2, None)),
             ("sr_debug_sqrt_mismatches", (0, 1, None)), ("sr_debug_log100_mismatches", (0, 1, None)),
             ("sr_debug_log100_mismatches", (0, (1 << 32) + 1, a)), ("sr_debug_mag10_mismatches", (0, 0, 1, None)),
             ("sr_debug_mag10_mismatches", (2, 0, 1, a)), ("sr_debug_mag10_mismatches", (0, 0, 16419 ** 2 + 1, a)),
             ("sr_debug_mag10_mismatches", (1, 0, (1 << 32) + 1, a)),
             ("sr_noise_atap_batch_dev", (None, U, 1, 2400, a)), ("sr_vad_batch_dev", (a, U, 1, U, a, None)),
             ("sr_mfcc_batch_dev", (a, U, 1, None, 2, a, a)), ("sr_dtw_batch_dev", (None, 1, 0, 0, a, a, a)),
             ("sr_recognise_batch_dev", (None, U, 1, 2400, C.byref(sr_b200.RecogOut())))]
    for fn, args in cases:
        l0 = h.launch_count()
        rc, err = _rc(h, fn, *args)
        assert rc == -1 and err, fn
        assert h.launch_count() == l0, fn


def test_zero_size_calls_do_nothing(h):
    o = C.byref(sr_b200.RecogOut())
    cases = [("sr_noise_atap_batch", (None, U, 0, 2400, None)), ("sr_vad_batch", (None, U, 0, U, None, None)),
             ("sr_mfcc_batch", (None, U, 0, None, 2, None, None)), ("sr_dtw_batch", (None, 0, 0, 0, None, None, None)),
             ("sr_recognise_batch", (None, U, 0, 2400, o)), ("sr_enrol_batch", (None, U, 0, 2400, None, 4096, None)),
             ("sr_get_mdl_batch", (None, None, 0, None, None)), ("sr_fft_mag_batch", (None, 160, 0, None)),
             ("sr_fft_raw_batch", (None, 0, None)), ("sr_get_dis_batch", (None, None, 0, None)),
             ("sr_debug_fft_raw_n", (None, 256, 0, None)),
             ("sr_dtw_limit_batch", (None, None, None, None, 0, None)),
             ("sr_dtw_batch_dev", (None, 0, 0, 0, None, None, None)), ("sr_recognise_batch_dev", (None, U, 0, 2400, o)),
             # checks that come after the early return
             ("sr_noise_atap_batch", (None, 70000, 0, 2400, None)), ("sr_vad_batch", (None, 70000, 0, 80000, None, None)),
             ("sr_dtw_batch", (None, 0, sr_b200.DTW_BAND, -1, None, None, None)),
             ("sr_dtw_batch_dev", (None, 0, sr_b200.DTW_BAND, -1, None, None, None))]
    for fn, args in cases:
        h.timing_collect()
        l0 = h.launch_count()
        assert _rc(h, fn, *args)[0] == 0, fn
        assert h.launch_count() == l0 and h.timing_collect() == [], fn
    for fn, args in [("sr_noise_atap_batch_dev", (None, U, 0, 2400, None)), ("sr_vad_batch_dev", (None, U, 0, U, None, None)),
                     ("sr_mfcc_batch_dev", (None, U, 0, None, 2, None, None))]:
        l0 = h.launch_count()
        assert _rc(h, fn, *args)[0] == 0, fn
        assert h.launch_count() == l0, fn
    h.timing_collect()


def test_checks_before_the_zero_size_early_return(h):
    a = np.zeros(64, np.uint8).ctypes.data
    o = C.byref(sr_b200.RecogOut())
    cases = [("sr_mfcc_batch", (None, U, 0, None, 1, None, None)),                 # seg_stride < 2
             ("sr_mfcc_batch_dev", (None, U, 0, None, 1, None, None)),
             ("sr_mfcc_batch_dev", (None, U, 0, None, 2, None, a + 2)),              # ftr not 4-byte aligned
             ("sr_noise_atap_batch_dev", (None, 70000, 0, 2400, None)),             # U > 65535
             ("sr_vad_batch_dev", (None, U, 0, U + 1, None, None)),                 # buf_len > U
             ("sr_dtw_batch_dev", (a + 2, 0, 0, 0, None, None, None)),              # in not 4-byte aligned
             ("sr_recognise_batch", (None, U, 0, U + 1, o)),                        # n_len > U
             ("sr_recognise_batch", (None, 70000, 0, 2400, o)),
             ("sr_recognise_batch", (None, U, 0, 2400, None)),                      # o == NULL
             ("sr_recognise_batch_dev", (None, U, 0, U + 1, o)),
             ("sr_enrol_batch", (None, U, 0, 2400, None, 2048, None)),              # slot_stride < sizeof(v_ftr_tag)
             ("sr_enrol_batch", (None, U, 0, 2400, None, 4098, None)),              # slot_stride % 4 != 0
             ("sr_fft_mag_batch", (None, 1025, 0, None)),                           # len > SR_FFT_POINT
             ("sr_debug_fft_raw_n", (None, 512, 0, None)),                          # N not 256 or 1024
             ("sr_debug_unpack12", (None, 0, None)),                                # NULL even when n == 0
             ("sr_debug_unpack12", (a, 3, a))]                                      # odd n
    for fn, args in cases:
        l0 = h.launch_count()
        rc, err = _rc(h, fn, *args)
        assert rc == -1 and err, fn
        assert h.launch_count() == l0, fn
    assert _rc(h, "sr_debug_unpack12", a, 0, a)[0] == 0


def test_band_radius_is_checked_when_the_band_scan_runs(h, data):
    ftr = data["ftr"]
    B = ftr.shape[0]
    s, bi, bd = np.zeros((B, T), np.uint32), np.zeros(B, np.uint32), np.zeros(B, np.uint32)
    rc, err = _rc(h, "sr_dtw_batch", ftr.ctypes.data, B, sr_b200.DTW_BAND, -1, s.ctypes.data, bi.ctypes.data, bd.ctypes.data)
    assert rc == -1 and err
    h.sync()
    h.timing_collect()


# ---- workspaces: growth and reuse never change a result --------------------------------------------------------------
def _calls():
    def pcm(n):
        return sr_b200.synth_pcm_host(n, U, 0x6A6A0000)

    def ftr(n):
        return sr_b200.synth_ftr_host(n, 0x6B6B0000, 20, 119).view(sr_b200.FTR_DTYPE).reshape(n).copy()

    def front(h, n):
        p = pcm(n)
        a = h.noise_atap(p, 2400)
        s = h.vad(p, a)
        return a, s, h.mfcc(p, s, a)

    def dtw(h, n):
        return h.dtw(ftr(n)) + h.dtw(ftr(n), sr_b200.DTW_BAND, 6)

    def recognise(h, n):
        return tuple(h.recognise(pcm(n), 2400).values())

    def get_mdl(h, n):
        f = ftr(n)
        return h.get_mdl(f, np.ascontiguousarray(f[::-1]))

    def fft(h, n):
        rng = np.random.default_rng(n)
        return (h.fft_mag(rng.integers(-2000, 2000, (n, 200)).astype(np.int16)),
                h.fft_raw(rng.integers(0, 1 << 32, (n, 1024), dtype=np.uint32)))

    def get_dis(h, n):
        rng = np.random.default_rng(n)
        a, b = (rng.integers(-3000, 3000, (n, 12)).astype(np.int16) for _ in range(2))
        return (h.get_dis(a, b),)

    def dtw_limit(h, n):
        rng = np.random.default_rng(n)
        x, y, i, m = (rng.integers(1, 120, n).astype(np.uint16) for _ in range(4))
        out = np.zeros(n, np.uint8)
        assert _rc(h, "sr_dtw_limit_batch", *[v.ctypes.data for v in (x, y, i, m)], n, out.ctypes.data)[0] == 0
        return (out,)

    def unpack12(h, n):
        return (h.unpack12(np.random.default_rng(n).integers(0, 256, 3 * n, dtype=np.uint8), 2 * n),)

    def enrol(h, n):
        return h.enrol(pcm(n), 2400)

    return {f.__name__: f for f in (front, dtw, recognise, get_mdl, fft, get_dis, dtw_limit, unpack12, enrol)}


def _equal(x, y):
    """equal outputs; of feature sets only save_sign, frm_num and the frm_num rows are results"""
    assert len(x) == len(y)
    for a, b in zip(x, y):
        if np.asarray(a).dtype == sr_b200.FTR_DTYPE:
            assert np.array_equal(a["save_sign"], b["save_sign"]) and ob.ftr_equal(a, b)
        else:
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("call", sorted(_calls()))
def test_workspace_growth_keeps_results(call):
    f = _calls()[call]
    small, large = 5, 300
    grow, shrink = _handle(), _handle()
    a_small, a_large = f(grow, small), f(grow, large)         # fresh handle -> small, then the workspaces grow
    b_large, b_small = f(shrink, large), f(shrink, small)     # fresh handle -> large, then a smaller call reuses them
    _equal(a_small, b_small)
    _equal(a_large, b_large)
    grow.close(); shrink.close()


# ---- reference-named drop-ins: the failure sentinels with a device present -------------------------------------------
def test_drop_in_sentinels_on_bad_arguments():
    L = sr_b200.lib()
    a = np.zeros(12, np.int16)
    f = np.zeros(2, sr_b200.FTR_DTYPE)
    assert L.get_dis(None, a.ctypes.data_as(C.c_void_p)) == sr_b200.DIS_ERR
    assert L.dtw(f[0:1].ctypes.data_as(C.c_void_p), None) == sr_b200.DIS_ERR
    assert not L.fft(None, 12) and not L.fft(a.ctypes.data_as(C.c_void_p), 1025)
    atap = np.zeros(1, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 7
    L.noise_atap(None, 2400, atap.ctypes.data_as(C.c_void_p))
    assert (atap["mid_val"] == 7).all()
    vv = (sr_b200.ValidTag * 3)(*[sr_b200.ValidTag(8, 16)] * 3)
    L.VAD(None, 100, vv, atap.ctypes.data_as(C.c_void_p))
    assert all(v.start is None and v.end is None for v in vv)
    f["frm_num"] = 9
    L.get_mfcc(None, f[0:1].ctypes.data_as(C.c_void_p), atap.ctypes.data_as(C.c_void_p))
    assert f["frm_num"][0] == 0
    # dtw() scores against a one-slot bank of its own: the same as a handle holding that template
    g = sr_b200.synth_ftr_host(2, 0x1D1D, 40, 90).view(sr_b200.FTR_DTYPE).reshape(2).copy()
    d = L.dtw(g[0:1].ctypes.data_as(C.c_void_p), g[1:2].ctypes.data_as(C.c_void_p))
    h = sr_b200.Handle(0)
    h.set_bank(sr_b200.make_bank(g[1:2], 2860), 1, 2860)
    assert d == h.dtw(g[0:1])[0][0, 0]
    h.close()
