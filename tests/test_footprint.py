"""The footprint of the entry points: which bytes of the caller's buffers a call writes, and which input bytes its results
may depend on. The value tests compare the frm_num rows of outputs the binding allocated itself, from inputs that are
clean up to their edges; here outputs sit in pattern- or sentinel-filled memory and inputs carry poison outside the bytes
a call may read. Every test requires (a) results equal to the oracle (or the plain references) on the clean inputs and
(b) every byte outside the documented write set unchanged.

Write sets (include/speech_recog.h): ftr -- frm_num and rows < frm_num of each struct, host calls included (MFCC.C
never writes save_sign); seg_off [B][3][2]; atap [B], only when n_len % 240 == 0; score [B][n_slot]; best_idx,
best_dis, cmd, status [B]; get_mdl -- frm_num and rows < frm_num of accepted pairs, rejected pairs untouched; the
long-form calls (include/sr_long.h) -- n_segs [B], atap [B] only when n_len % 240 == 0 and n_len <= lens[b], segment
slots and records k < min(n_segs[b], max_segs).
Read sets: MFCC samples [start - 1, end), [start, end) when start == 0; noise_atap / VAD samples < n_len / buf_len;
features rows < frm_num (the greedy walk: rows < max(frm_num + 1, 2)); banks the v_ftr_tag of the slots a scan walks;
stream chunks lens[s] / chunk_len samples per row, up to max_samples per stream; long-form recordings lens[b] samples.

Guards and poison lie inside the allocation they surround: no access made here leaves an allocation."""
import ctypes as C

import numpy as np
import pytest

import oracle_ext as ox
import oracle_bind as ob
import sr_b200

pytestmark = pytest.mark.gpu

FTR = sr_b200.FTR_DTYPE
FB = sr_b200.FTR_BYTES
P8, Q8 = 0xA5, 0x3C          # P: what earlier calls leave in the handle's workspaces; Q: what the caller's structs hold
SENT = 0xC7                  # sentinel around device outputs
GUARD = 4096
OFF = GUARD + 4              # outputs start 4-byte but not 16-byte aligned
T = 40                       # templates: more than one 32-slot tile
FULL = np.array([32767, -32768], np.int16)


@pytest.fixture(scope="module")
def ora():
    return ob.best_oracle()


@pytest.fixture(scope="module")
def bank():
    h = sr_b200.Handle(0)
    b, st = h.enrol(sr_b200.synth_pcm_host(T, 8000, 0x7E3A0000), 2400)
    h.close()
    assert (st == 0).sum() >= T - 2
    return b


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _handle(bank=None, geom=0):
    h = sr_b200.Handle(0)
    h.set_transport(0)
    h.set_geometry(geom)
    if bank is not None:
        h.set_bank(bank, T, 4096)
    return h


# ---- feature structs ------------------------------------------------------------------------------------------------
def _filled(n, byte):
    f = np.zeros(n, FTR)
    f.view(np.uint8)[:] = byte
    return f


def _prime(h, n):
    """sr_dtw_batch of n structs whose every row is pattern P: the handle's feature workspace then holds P, the bytes a
    copy-back of rows the kernels never wrote would hand out"""
    f = _filled(n, P8)
    f["frm_num"] = 40
    h.dtw(f, want_score=False)


def _written(ftr):
    """[n, 2860] mask of the bytes get_mfcc may write: frm_num and rows < frm_num"""
    n = ftr["frm_num"].astype(np.int64)
    col = np.arange(FB)[None, :]
    return ((col >= 2) & (col < 4)) | ((col >= 4) & (col < 4 + 24 * n[:, None]))


def _check_ftr(got, want, fill, what=""):
    """got holds want's frm_num and frm_num rows, and every other byte is still `fill`"""
    assert ob.ftr_equal(got, want), what
    raw = got.view(np.uint8).reshape(-1, FB)
    bad = ~_written(got) & (raw != fill)
    if bad.any():
        u = int(np.flatnonzero(bad.any(axis=1))[0])
        b = int(np.flatnonzero(bad[u])[0])
        raise AssertionError("%s: %d structs changed outside frm_num and its rows; struct %d (frm_num %d): byte %d (row %d) "
                             "is 0x%02x, the caller's was 0x%02x" % (what, int(bad.any(axis=1).sum()), u,
                                                                    got["frm_num"][u], b, (b - 4) // 24, raw[u, b], fill))


def _segments(rng, B, U, frame):
    """B segments of U-sample rows, starts >= 1: the frame-count edges (0, 1, 119, 120 frames), NULL, segments that end
    at U, and random lengths"""
    f119, f120 = frame + 80 * 118, frame + 80 * 119
    edges = [0, frame - 1, frame, frame + 1, f119, f119 + 79, f120, f120 + 500]
    ln = np.where(np.arange(B) < len(edges), np.resize(edges, B), frame + rng.integers(0, 80 * 119, B))
    st = 1 + rng.integers(0, U - ln)
    st[len(edges)::7] = U - ln[len(edges)::7]                      # every 7th ends at the last sample of its row
    seg = np.stack([st, st + ln], 1).astype(np.uint32)
    seg[len(edges) + 3::11] = ob.NULL
    return seg


def _mfcc_want(ora, pcm, seg, atap, geom_b):
    B = len(pcm)
    want = np.zeros(B, FTR)
    ok = (seg != ob.NULL).all(axis=1)
    f = ob.port().mfcc_geom_b_batch if geom_b else ora.mfcc_batch
    want[ok] = f(pcm[ok], seg[ok], atap[ok])
    return want


def _front(pcm, U):
    h = _handle()
    atap = h.noise_atap(pcm, 2400)
    h.close()
    return atap


# ---- writes of the host-buffer calls --------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [0, 1], ids=["ref", "geom_b"])
def test_mfcc_batch_writes_only_frm_num_and_its_rows(ora, geom):
    """a workspace that last held another call's rows must not reach the caller: save_sign and every row >= frm_num of
    each struct come back as the caller passed them (pattern Q, not the primed P), rejected segments included"""
    B, U = 300, 12000
    pcm = sr_b200.synth_pcm_host(B, U, 0x3F00 + geom, 2)
    seg = _segments(np.random.default_rng(3 + geom), B, U, 200 if geom else 160)
    atap = _front(pcm, U)
    want = _mfcc_want(ora, pcm, seg, atap, geom == 1)
    assert (want["frm_num"] == 0).sum() >= 10 and (want["frm_num"] == 1).any() and (want["frm_num"] == 119).any()
    h = _handle(geom=geom)
    _prime(h, B)
    _check_ftr(h.mfcc(pcm, seg, atap, ftr=_filled(B, Q8)), want, Q8, "sr_mfcc_batch")
    h.close()


@pytest.mark.parametrize("transport", [0, 1], ids=["plain", "packed"])
def test_recognise_batch_writes_only_frm_num_and_its_rows(ora, bank, transport):
    """sr_recognise_batch with ftr requested over four 32 MB chunks, plain and 12-bit packed"""
    U, B = 8000, 3 * 2096 + 8
    pcm = sr_b200.synth_pcm_host(B, U, 0x2C2D)
    h = _handle(bank)
    h.set_transport(transport)
    for _ in range(3):                                              # packed: the caller's thread may outrun the packers
        _prime(h, B)
        out = sr_b200._recog_arrays(B, T, ("ftr", "status", "best_idx"))
        out["ftr"] = _filled(B, Q8)
        h._ck(sr_b200.lib().sr_recognise_batch(h._h, sr_b200._p(pcm), U, B, 2400, C.byref(sr_b200._recog_out(out))))
        packed, plain, _ = h.transport_stats()
        assert packed + plain == 4 and (transport == 1 or packed == 0)
        if transport == 0 or packed >= 1:
            break
    else:
        pytest.skip("no chunk went packed in three calls: this host has no packer pool (too few CPUs)")
    assert (out["status"] == 0).any()
    rows = np.r_[0:8, 2090:2100, 4188:4196, B - 8:B]                # the ends of every chunk
    want = ob.recognise_pinned(ora, pcm[rows], 2400, bank, T, 4096)
    _check_ftr(out["ftr"][rows], want["ftr"], Q8, "sr_recognise_batch at the chunk edges")
    assert np.array_equal(out["best_idx"][rows], want["best_idx"])
    _check_ftr(out["ftr"], out["ftr"], Q8, "sr_recognise_batch")
    h.close()


def test_recognise_multi_writes_only_frm_num_and_its_rows(ora, bank):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    U, B = 8000, 203
    pcm = sr_b200.synth_pcm_host(B, U, 0x2C2E)
    hs = [sr_b200.Handle(d) for d in range(torch.cuda.device_count())]
    for h in hs:
        h.set_transport(0)
        h.set_bank(bank, T, 4096)
        _prime(h, B)
    out = sr_b200._recog_arrays(B, T, ("ftr", "best_idx"))
    out["ftr"] = _filled(B, Q8)
    arr = (C.c_void_p * len(hs))(*[h._h for h in hs])
    assert sr_b200.lib().sr_recognise_batch_multi(arr, len(hs), sr_b200._p(pcm), U, B, 2400,
                                                  C.byref(sr_b200._recog_out(out))) == 0
    want = ob.recognise_pinned(ora, pcm, 2400, bank, T, 4096)
    _check_ftr(out["ftr"], want["ftr"], Q8, "sr_recognise_batch_multi")
    for h in hs:
        h.close()


def test_drop_in_get_mfcc_writes_only_frm_num_and_its_rows(ora):
    """get_mfcc on the default handle, after dtw() left pattern P in its workspace: 1, 119, 120 frames and a typical
    segment"""
    L = sr_b200.lib()
    pcm = sr_b200.synth_pcm_host(1, 12000, 0x6161, 2)[0]
    atap = _front(pcm[None, :], 12000)
    for ln in (160, 160 + 80 * 118, 160 + 80 * 119, 3000):
        p = _filled(2, P8)
        p["frm_num"] = 40
        L.dtw(p[0:1].ctypes.data_as(C.c_void_p), p[1:2].ctypes.data_as(C.c_void_p))
        st = 700
        vt = sr_b200.ValidTag(pcm.ctypes.data + 2 * st, pcm.ctypes.data + 2 * (st + ln))
        got = _filled(1, Q8)
        L.get_mfcc(C.byref(vt), got.ctypes.data_as(C.c_void_p), atap.ctypes.data_as(C.c_void_p))
        want = ora.mfcc_batch(pcm[None, :], np.array([[st, st + ln]], np.uint32), atap)
        assert (want["frm_num"][0] == 0) == (ln > 160 + 80 * 118)
        _check_ftr(got, want, Q8, "get_mfcc of %d samples" % ln)


def test_get_mdl_keeps_rows_past_the_new_frm_num():
    rng = np.random.default_rng(0x6D)
    n = 64
    fi = [rng.integers(-3000, 3001, (int(rng.integers(20, 60)), 12)) for _ in range(n)]
    fm = [rng.integers(-3000, 3001, (int(rng.integers(20, 60)), 12)) for _ in range(n)]
    fm[5] = rng.integers(-3000, 3001, (2 * len(fi[5]) + 1, 12))  # the 2:1 guard rejects the pair
    from test_extension_refs import _ftr
    a, b = _ftr(fi), _ftr(fm)
    want, wdis = ob.port().get_mdl(a, b)
    h = _handle()
    _prime(h, n)
    got, dis = h.get_mdl(a, b, mdl=_filled(n, Q8))
    assert np.array_equal(dis, wdis) and wdis[5] == sr_b200.DIS_ERR
    ok = dis != sr_b200.DIS_ERR
    _check_ftr(got[ok], want[ok], Q8, "sr_get_mdl_batch")
    assert (got[~ok].view(np.uint8) == Q8).all()
    h.close()


def test_path_and_average_write_every_output_byte():
    """sr_dtw_path_batch and sr_average_bank called with outputs prefilled with two different patterns return the same
    bytes, those of the oracle: no byte of path, path_len, dis, bank_out, score or anchor is left as the caller had it"""
    from test_dp_align import _random_groups
    L = sr_b200.lib()
    h = _handle()
    rng = np.random.default_rng(0x9A)
    n = 150
    from test_extension_refs import _ftr
    a = _ftr([rng.integers(-3000, 3001, (int(rng.integers(1, 120)), 12)) for _ in range(n)])
    b = _ftr([rng.integers(-3000, 3001, (int(rng.integers(1, 120)), 12)) for _ in range(n)])
    want = ox.align().dtw_path(a, b, 10)
    for fill in (P8, Q8):
        path, plen, dis = (np.full(s, fill, np.uint8) for s in (n * 237 * 2, n * 4, n * 4))
        assert L.sr_dtw_path_batch(h._h, a.ctypes.data, b.ctypes.data, n, 10, path.ctypes.data, plen.ctypes.data,
                                   dis.ctypes.data) == 0
        assert np.array_equal(dis.view(np.uint32), want[0]) and np.array_equal(plen.view(np.uint32), want[2])
        assert np.array_equal(path.reshape(n, 237, 2), want[1])
    K, G, stride = 4, 40, 4096
    bk = _random_groups(rng, G, K, stride, fmin=5, fmax=60)
    want = ox.align().average_bank(bk, stride, K, 10, 2)
    for fill in (P8, Q8):
        out, score, anchor = (np.full(s, fill, np.uint8) for s in (G * K * stride, G * K * 4, G * 4))
        assert L.sr_average_bank(h._h, bk.ctypes.data, stride, K, G, 10, 2, out.ctypes.data, score.ctypes.data,
                                 anchor.ctypes.data) == 0
        assert np.array_equal(out.reshape(G * K, stride), want[0])
        assert np.array_equal(score.view(np.uint32).reshape(G, K), want[1])
        assert np.array_equal(anchor.view(np.uint32), want[2])
    h.close()


# ---- device pointers: guarded outputs, unchanged inputs --------------------------------------------------------------
class Dev:
    """a device buffer holding `nbytes` at byte offset `off` with `fill` in every other byte of the allocation (at least
    GUARD bytes on each side)"""

    def __init__(self, nbytes, fill=SENT, off=OFF, data=None):
        import torch
        self.off, self.n, self.fill = off, nbytes, fill
        self.t = torch.full((off + nbytes + GUARD + 12,), fill, dtype=torch.uint8, device="cuda:0")
        if data is not None:
            raw = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
            assert raw.size == nbytes
            self.t[off:off + nbytes] = torch.from_numpy(raw.copy()).to("cuda:0")
        torch.cuda.synchronize()
        self.before = self.all()

    @property
    def ptr(self):
        return self.t.data_ptr() + self.off

    def all(self):
        import torch
        torch.cuda.synchronize()
        return self.t.cpu().numpy()

    def body(self):
        return self.all()[self.off:self.off + self.n]

    def unchanged(self, what):
        assert np.array_equal(self.all(), self.before), "%s: input bytes changed" % what

    def check(self, want, mask=None, what=""):
        """the guards still hold the fill; the body equals want where mask (default: everywhere) and the fill elsewhere"""
        a = self.all()
        out = np.r_[0:self.off, self.off + self.n:a.size]
        assert (a[out] == self.fill).all(), "%s: %d guard bytes changed" % (what, int((a[out] != self.fill).sum()))
        body, want = a[self.off:self.off + self.n], np.ascontiguousarray(want).view(np.uint8).reshape(-1)
        mask = np.ones(self.n, bool) if mask is None else mask.reshape(-1)
        assert np.array_equal(body[mask], want[mask]), "%s: wrong values" % what
        assert (body[~mask] == self.fill).all(), "%s: %d bytes outside the write set changed" % (what, int((body[~mask] != self.fill).sum()))


def _pcm_dev(pcm, phase=0, poison=None):
    """PCM rows at a 16-byte boundary + phase bytes, the rest of the allocation `poison` (u16 pattern) or SENT"""
    d = Dev(pcm.nbytes, off=GUARD + phase, data=pcm)
    if poison is not None:
        import torch
        a = d.all()
        pv = np.resize(np.asarray(poison, np.uint16), (a.size + 1) // 2).view(np.uint8)[:a.size]
        a[:d.off], a[d.off + d.n:] = pv[:d.off], pv[d.off + d.n:]
        d.t.copy_(torch.from_numpy(a))
        d.before = d.all()
    return d


def test_front_end_dev_writes_and_reads(bank):
    """sr_noise_atap_batch_dev, sr_vad_batch_dev and sr_mfcc_batch_dev (both geometries) at batch sizes on both sides of
    the persistent grids' hand-out units: VAD SMs x 20 warps, MFCC SMs CTAs, GEOM_B SMs x 4 CTAs. The values are those of
    the host-buffer calls on the same handle, which the parity tests hold to the oracle."""
    n = _sms()
    U = 8000
    for B in (1, n - 1, n + 1, 4 * n - 1, 4 * n + 1, 20 * n - 1, 20 * n + 1):
        pcm = sr_b200.synth_pcm_host(B, U, 0x1357 + B)
        h = _handle()
        atap = h.noise_atap(pcm, 2400)
        seg = h.vad(pcm, atap)
        pd = _pcm_dev(pcm, 2, poison=[0xFFFF, 0])
        for n_len in (2400, 2401):
            at = Dev(B * 12)
            h.noise_atap_dev(pd.ptr, U, B, n_len, at.ptr)
            h.sync()
            at.check(atap, None if n_len == 2400 else np.zeros(B * 12, bool), "noise_atap_dev n_len %d, B %d" % (n_len, B))
        ad = Dev(B * 12, data=atap)
        sg = Dev(B * 24)
        h.vad_dev(pd.ptr, U, B, U, ad.ptr, sg.ptr)
        h.sync()
        sg.check(seg, what="vad_dev B %d" % B)
        ad.unchanged("vad_dev atap")
        sd = Dev(B * 24, data=seg)
        for geom in (0, 1):
            h.set_geometry(geom)
            want = h.mfcc(pcm, seg, atap)
            ft = Dev(B * FB)
            h.mfcc_dev(pd.ptr, U, B, sd.ptr, 6, ad.ptr, ft.ptr)
            h.sync()
            ft.check(want, _written(want), "mfcc_dev geom %d B %d" % (geom, B))
        h.set_geometry(0)
        pd.unchanged("pcm")
        ad.unchanged("atap")
        sd.unchanged("seg")
        h.close()


def _lane_utts(Tt):
    """utterances one CTA takes per pass of the lane-packed scans (dtw_kernel, dtw_band_thread_kernel<10>) on a tile of
    Tt templates: G * NU of the lane plan plan_lanes (sr_dtw.cu) picks, the busiest (Wg, NU, G) within shared memory"""
    slot = 119 * 24 + 120 * 4                                       # kSlotBytes: rows + squared norms
    slots_max = (224 * 1024 - Tt * slot - 256 - 512) // slot
    best, pick = -1.0, 0
    for wg in range(1, 9):
        nu = 32 * wg // Tt
        g = min(32 // wg, slots_max // nu if nu else 0, 15 if wg > 1 else 32)
        if nu < 1 or g < 1:
            continue
        util = (nu * Tt / (32.0 * wg)) * (g * wg / 32.0)
        if util > best + 1e-9:
            best, pick = util, g * nu
    return pick


def _scan_units(scan, n):
    """the hand-out units of a template scan over T templates on n SMs: utterances one pass of each launch's grid covers
    before its CTAs stride on (grid_rows in sr_dtw_core.cuh). The lane-packed and dynamic scans launch once for the full
    32-template tiles and once for the remainder tile; the warp-per-pair band kernels (r != 10) launch all tiles at once,
    16 warps per CTA"""
    full, rem = T // 32, T % 32
    if scan in ("band7", "band16"):
        return [(n // (full + (rem > 0))) * 16]
    per = {"greedy": _lane_utts, "band10": _lane_utts, "greedy_dyn": lambda Tt: 1}[scan]
    return ([(n // full) * per(32)] if full else []) + ([n * per(rem)] if rem else [])


def _sizes(units):
    """batch sizes just below and just past each unit and its double"""
    return sorted({1, 33} | {k * u + d for u in units for k in (1, 2) for d in (-1, 1)})


@pytest.mark.parametrize("scan", ["greedy", "greedy_dyn", "band7", "band10", "band16"])
def test_dtw_dev_writes_and_reads(ora, bank, scan):
    """sr_dtw_batch_dev: score [B][T], best_idx, best_dis at 4-byte-aligned offsets, nothing past them (settles that no
    scan writes the word after score), against a bank set with sr_set_bank_dev; inputs and bank unchanged. Batch sizes
    on both sides of one and two passes of every launch's grid (H100, T = 40: the greedy and r = 10 scans take 32
    utterances per CTA on the 32-template tile and 60 on the 8-template one, 4 224 and 7 920 per pass; the dynamic greedy
    scan one per CTA; r = 7 and 16 one per warp, 66 CTA rows x 16); a sample equals the oracle."""
    n = _sms()
    flags, r = (0, 0) if scan.startswith("greedy") else (sr_b200.DTW_BAND, int(scan[4:]))
    h = _handle()
    h.set_dtw_variant(1 if scan == "greedy_dyn" else 0)
    bd = Dev(bank.nbytes, data=bank)
    h.set_bank_dev(bd.ptr, T, 4096)
    for B in _sizes(_scan_units(scan, n)):
        f = sr_b200.synth_ftr_host(B, 0x5150 + B, 1, 119).view(FTR).reshape(B).copy()
        fd = Dev(f.nbytes, data=f)
        sc, bi, bs = Dev(B * T * 4), Dev(B * 4), Dev(B * 4)
        h.dtw_dev(fd.ptr, B, flags, r, sc.ptr, bi.ptr, bs.ptr)
        h.sync()
        s = np.random.default_rng(B).choice(B, min(B, 48), replace=False)
        o = ora if not flags else ob.port()
        want, _ = o.dtw_batch(np.ascontiguousarray(f[s]), bank, T, 4096, band_r=r if flags else -1)
        got = sc.body().view(np.uint32).reshape(B, T)
        assert np.array_equal(got[s], want), (scan, B)
        key = (got.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)
        sc.check(got, what="score")
        bi.check((key.min(1) & 0xFFFFFFFF).astype(np.uint32), what="best_idx")
        bs.check((key.min(1) >> np.uint64(32)).astype(np.uint32), what="best_dis")
        fd.unchanged("ftr in")
    bd.unchanged("bank")
    h.close()


def test_recognise_dev_writes_and_reads(bank):
    """sr_recognise_batch_dev into guarded outputs, past one pass of the VAD grid (SMs x 20 warps) and of each greedy scan
    launch (_scan_units); the values are those of sr_recognise_batch on the same handle, which the parity tests hold to
    the oracle"""
    n = _sms()
    U = 8000
    h = _handle()
    bd = Dev(bank.nbytes, data=bank)
    h.set_bank_dev(bd.ptr, T, 4096)
    for B in sorted({1, n + 1, 20 * n - 1, 20 * n + 1} | {u + 1 for u in _scan_units("greedy", n)}):
        pcm = sr_b200.synth_pcm_host(B, U, 0x2468 + B)
        h.set_bank(bank, T, 4096)
        want = h.recognise(pcm, 2400)
        h.set_bank_dev(bd.ptr, T, 4096)
        pd = _pcm_dev(pcm, 6, poison=[0xFFFF, 0])
        size = {"atap": 12, "seg_off": 24, "ftr": FB, "score": 4 * T, "best_idx": 4, "best_dis": 4, "cmd": 4, "status": 1}
        o = {k: Dev(B * v) for k, v in size.items()}
        h.recognise_dev(pd.ptr, U, B, 2400, **{k: v.ptr for k, v in o.items()})
        h.sync()
        for k, d in o.items():
            d.check(want[k], _written(want[k]) if k == "ftr" else None, "recognise_dev %s B %d" % (k, B))
        pd.unchanged("pcm")
    bd.unchanged("bank")
    h.close()


# ---- the long-form calls (include/sr_long.h) -----------------------------------------------------------------------------
def _long_slots(n_segs, max_segs, nbytes):
    """[B * max_segs * nbytes] mask of the slots a long-form call writes: k < min(n_segs[b], max_segs)"""
    k = np.arange(max_segs)[None, :] < np.minimum(n_segs, max_segs)[:, None]
    return np.repeat(k.reshape(-1), nbytes)


def test_long_dev_writes_and_reads(bank):
    """sr_vad_long_batch_dev and sr_recognise_long_batch_dev into outputs 4 bytes past a 16-byte boundary between
    sentinels, on a handle whose workspaces an earlier, larger call left full (more recordings, more segments, another U):
    atap is written only for rows with n_len % 240 == 0 and n_len <= lens[b]; segment slots and records only below
    min(n_segs, max_segs); lens[b] > U reads as U; loud band-crossing poison past lens[b] and after the last row changes
    nothing. The host calls on the same handle equal those of a fresh handle and the oracle."""
    lo, port = ox.long_oracle(), ob.port()
    B, U = 8, 30011
    lens = np.array([2399, 2400, 2401, 0, U, U + 1, 0xFFFFFFFF, 20000], np.uint32)   # n_len - 1, n_len, n_len + 1, 0, >= U
    eff = np.minimum(lens, U)
    pcm = ox.synth_long(B, U, 0x1A5)
    for b in range(B):
        pcm[b, eff[b]:] = np.where(np.arange(U - eff[b]) % 2, 4095, 0)
    atap0 = np.zeros(B, ob.ATAP_DTYPE)
    atap0["mid_val"], atap0["n_thl"], atap0["z_thl"], atap0["s_thl"] = 2000 + np.arange(B), 40, 2, 3000
    h = _handle(bank)
    stale = ox.synth_long(12, 50000, 0x1A6)
    assert h.recognise_long_batch(stale, 64, 2400)["n_segs"].sum() > 40
    for n_len, ms, phase in ((2400, 3, 0), (2400, 64, 2), (2401, 64, 0), (2400, 0, 2)):
        what = "n_len %d max_segs %d phase %d" % (n_len, ms, phase)
        want = ox.recognise_long(lo, port, pcm, n_len, bank, T, 4096, ms, eff, atap=atap0)
        want_n, want_seg = lo.vad_long(pcm, want["atap"], ms, eff)
        assert want["n_segs"].tolist() == want_n.tolist()
        if n_len == 2400:
            assert [want["atap"][b].tobytes() == atap0[b].tobytes() for b in range(4)] == [True, False, False, True]
        pd, ld = _pcm_dev(pcm, phase, poison=[4095, 0]), Dev(lens.nbytes, data=lens)
        ad, nd, sd = Dev(atap0.nbytes, data=atap0), Dev(B * 4), Dev(B * ms * 8)
        h.vad_long_batch_dev(pd.ptr, U, B, ld.ptr, n_len, ms, ad.ptr, nd.ptr, sd.ptr if ms else None)
        h.sync()
        ad.check(want["atap"], what=what + " vad atap")
        nd.check(want_n, what=what + " n_segs")
        sd.check(want_seg, _long_slots(want_n, ms, 8), what + " seg_off")
        ad, nd, rd = Dev(atap0.nbytes, data=atap0), Dev(B * 4), Dev(B * ms * 28)
        h.recognise_long_batch_dev(pd.ptr, U, B, ld.ptr, n_len, ms, ad.ptr, nd.ptr, rd.ptr if ms else None)
        h.sync()
        ad.check(want["atap"], what=what + " recognise atap")
        nd.check(want_n, what=what + " recognise n_segs")
        rd.check(want["segs"], _long_slots(want_n, ms, 28), what + " records")
        pd.unchanged("pcm")
        ld.unchanged("lens")
        assert (ms == 64 or (want_n > ms).any()) and (want["segs"]["status"] == 0).sum() >= min(ms, 3)
    # the host calls (lens <= U) after all of that, against a fresh handle and the oracle
    fresh = _handle(bank)
    try:
        for hh in (h, fresh):
            got = hh.recognise_long_batch(pcm, 5, 2400, eff, atap=atap0.copy())
            want = ox.recognise_long(lo, port, pcm, 2400, bank, T, 4096, 5, eff, atap=atap0)
            for k in ("atap", "n_segs", "segs"):
                assert got[k].tobytes() == want[k].tobytes(), k
            v = hh.vad_long_batch(pcm, 5, 2400, eff, atap=atap0.copy())
            assert v["n_segs"].tolist() == want["n_segs"].tolist()
            assert (v["seg_off"][..., 0] == want["segs"]["start"]).all() and (v["seg_off"][..., 1] == want["segs"]["end"]).all()
    finally:
        fresh.close()
        h.close()


# ---- reads: poison outside the read set changes no result -----------------------------------------------------------
def _poison_outside(pcm, seg, atap, pattern):
    """a copy of pcm with every sample outside [start - 1, end) ([start, end) when start == 0) replaced by pattern"""
    out = np.resize(np.asarray(pattern, np.uint16), pcm.size).reshape(pcm.shape).copy()
    for b, (s, e) in enumerate(seg):
        if s == ob.NULL:
            continue
        lo = max(int(s) - 1, 0)
        out[b, lo:e] = pcm[b, lo:e]
    return out


@pytest.mark.parametrize("geom", [0, 1], ids=["ref", "geom_b"])
def test_mfcc_reads_only_its_segment(ora, geom):
    """host and _dev forms: full-scale poison and alternation around mid_val outside every segment, the PCM 2, 6 and 14
    bytes past a 16-byte boundary with poison in the rest of its granules; segments at sample 0 and at the row's end"""
    B, U = 140, 12003
    pcm = sr_b200.synth_pcm_host(B, U, 0x7070 + geom, 2)
    seg = _segments(np.random.default_rng(7 + geom), B, U, 200 if geom else 160)
    z = np.arange(0, B, 9)
    z = z[seg[z, 0] != ob.NULL]
    seg[z, 1] -= seg[z, 0]
    seg[z, 0] = 0                                                   # starts at 0: x[-1] is mid_val
    seg[0] = [0, 2500]                                              # the poison before row 0 borders a read sample
    seg[B - 1] = [U - 2500, U]                                      # and the poison after row B - 1
    atap = _front(pcm, U)
    want = _mfcc_want(ora, ob.pinned_rows(pcm, atap), np.where(seg == ob.NULL, seg, seg + 1), atap, geom == 1)
    h = _handle(geom=geom)
    mid = int(atap["mid_val"][0])
    for pattern in ([0xFFFF, 0], [mid + 1500, mid - 1500]):
        bad = _poison_outside(pcm, seg, atap, pattern)
        assert ob.ftr_equal(h.mfcc(bad, seg, atap), want), pattern
        for phase in (2, 6, 14):
            pd, sd, ad, ft = _pcm_dev(bad, phase, poison=pattern), Dev(seg.nbytes, data=seg), Dev(atap.nbytes, data=atap), Dev(B * FB)
            h.mfcc_dev(pd.ptr, U, B, sd.ptr, 2, ad.ptr, ft.ptr)
            h.sync()
            ft.check(want, _written(want), "mfcc_dev phase %d" % phase)
    h.close()


def test_noise_atap_and_vad_read_only_their_window(ora):
    B, U = 64, 8000
    pcm = sr_b200.synth_pcm_host(B, U, 0x7171)
    h = _handle()
    for n_len, buf_len in ((2400, 6001), (4800, 8000), (2160, 3000)):
        want_a = np.concatenate([ora.noise_atap(pcm[b], n_len) for b in range(B)])
        want_s = np.stack([ora.vad(pcm[b], buf_len, want_a[b:b + 1]) for b in range(B)]).reshape(B, 3, 2)
        for pattern in ([0xFFFF, 0], [4095, 0, 0, 4095]):
            bad = pcm.copy()
            bad[:, n_len:] = np.resize(np.asarray(pattern, np.uint16), U - n_len)
            assert h.noise_atap(bad, n_len).tobytes() == want_a.tobytes()
            bad = pcm.copy()
            bad[:, buf_len:] = np.resize(np.asarray(pattern, np.uint16), U - buf_len)
            assert np.array_equal(h.vad(bad, want_a, buf_len), want_s)
    h.close()


def _poison_rows(f, first_row, sign=False):
    """a copy of features f with every row >= first_row[b] set to full-scale alternation (and save_sign, with sign)"""
    g = f.copy()
    m = g["mfcc_dat"].reshape(len(g), 119, 12)
    for b in range(len(g)):
        m[b, int(first_row[b]):] = np.resize(FULL, (119 - int(first_row[b]), 12))
    g["mfcc_dat"] = m.reshape(len(g), -1)
    if sign:
        g["save_sign"] = 0x5A5A
    return g


def _poison_bank(bank, stride, first_row, walked):
    """a copy of a bank with rows >= first_row and the slot padding [2860, stride) poisoned; slots not walked get every
    byte after their header poisoned"""
    b = bank.copy().reshape(-1, stride)
    pv = np.resize(FULL, (stride - 4) // 2).view(np.uint8)
    for t in range(len(b)):
        lo = 4 + 24 * int(first_row[t]) if walked[t] else 4
        b[t, lo:] = pv[lo - 4:]
    return b


def _ftr_set(rng, B):
    from test_extension_refs import _ftr
    lens = np.r_[[1, 2, 3, 59, 118, 119], rng.integers(1, 120, B - 6)]
    return _ftr([rng.integers(-3000, 3001, (int(n), 12)) for n in lens])


def _test_bank(rng, stride):
    """T slots: signed ones of 1..119 frames, then an unsigned, an erased and a frm_num 120 one"""
    from test_extension_refs import _ftr
    f = _ftr([rng.integers(-3000, 3001, (int(n), 12)) for n in np.r_[[1, 2, 119], rng.integers(1, 120, T - 3)]])
    bk = sr_b200.make_bank(f, stride)
    bk[T - 3, :2] = 0                                               # unsigned
    bk[T - 2] = 0xFF                                                # erased
    bk[T - 1, 2:4] = [120, 0]                                       # frm_num 120
    return bk


@pytest.mark.parametrize("scan", ["greedy", "band7", "band10", "band16"])
def test_dtw_reads_only_the_rows_it_walks(ora, scan):
    """inputs: rows >= max(frm_num + 1, 2) for the greedy walk, rows >= frm_num and save_sign for the band scans; bank:
    the same rows of signed slots, the slot padding, and under SR_DTW_CHECK_SIGN every byte after the header of an
    unsigned, erased or frm_num 120 slot. The greedy walk's input row frm_num is poisoned on its own: DTW.C:141-191 is a
    do-while whose first step evaluates get_dis on row 1 of both sets before any bound test, guarded only by dtw_limit,
    so for a 1-frame set the reference may read row frm_num (the stager loads rows < max(frm_num + 1, 2) to match it);
    there only kernel == oracle on the poisoned input is required."""
    rng = np.random.default_rng(0xD7)
    stride, B = 4096, 200
    band = scan != "greedy"
    r = int(scan[4:]) if band else -1
    o = ob.port() if band else ora
    f = _ftr_set(rng, B)
    bk = _test_bank(rng, stride)
    h = _handle()
    flags = (sr_b200.DTW_BAND if band else 0) | sr_b200.DTW_CHECK_SIGN
    fn = f["frm_num"].astype(int)
    tn = np.frombuffer(bk[:, 2:4].tobytes(), np.uint16).astype(int)
    walked = np.arange(T) < T - 3
    want, _ = o.dtw_batch(f, bk, T, stride, check_sign=1, band_r=r)
    want[:, T - 1] = sr_b200.DIS_ERR          # frm_num > 119 is never walked (its rows would lie past the struct)
    first_in = fn if band else np.maximum(fn + 1, 2)
    first_t = np.minimum(tn if band else np.maximum(tn + 1, 2), 119)
    bad_f = _poison_rows(f, np.minimum(first_in, 119), sign=band)
    bad_b = _poison_bank(bk, stride, first_t, walked)
    for ff, bb in ((f, bk), (bad_f, bk), (f, bad_b), (bad_f, bad_b)):
        h.set_bank(bb, T, stride)
        got, _, _ = h.dtw(ff, flags, max(r, 0))
        assert np.array_equal(got, want), scan
    if not band:                                                    # row frm_num itself: kernel == oracle
        edge = _poison_rows(f, np.minimum(fn, 119))
        h.set_bank(bk, T, stride)
        got, _, _ = h.dtw(edge, flags, 0)
        want, _ = ora.dtw_batch(edge, bk, T, stride, check_sign=1)
        want[:, T - 1] = sr_b200.DIS_ERR
        assert np.array_equal(got, want)
    h.close()


def test_path_and_average_read_only_member_rows():
    """sr_dtw_path_batch: rows >= frm_num and save_sign of both sides; sr_average_bank: rows >= frm_num and padding of
    member slots, every byte after the header of a non-member slot"""
    from test_dp_align import _random_groups
    rng = np.random.default_rng(0xA1)
    h = _handle()
    a, b = _ftr_set(rng, 120), _ftr_set(rng, 120)
    for r in (7, 10, 16):
        want = ox.align().dtw_path(a, b, r)
        bad_a = _poison_rows(a, a["frm_num"], sign=True)
        bad_b = _poison_rows(b, b["frm_num"], sign=True)
        for x, y in ((bad_a, b), (a, bad_b), (bad_a, bad_b)):
            got = h.dtw_path(x, y, r)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), r
    K, G, stride = 4, 30, 4096
    bk = _random_groups(rng, G, K, stride, fmin=3, fmax=80)
    hdr = np.frombuffer(bk[:, :4].tobytes(), np.uint16).reshape(-1, 2).astype(int)
    member = (hdr[:, 0] == sr_b200.SAVE_MASK) & (hdr[:, 1] >= 1) & (hdr[:, 1] <= 119)
    assert (~member).sum() >= 4
    want = ox.align().average_bank(bk, stride, K, 10, 2)
    got = h.average_bank(_poison_bank(bk, stride, np.where(member, hdr[:, 1], 0), member), stride, K, 10, 2)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    h.close()


# ---- streaming: samples past lens[s] / chunk_len / max_samples ------------------------------------------------------
def _events_key(evs):
    return sorted(tuple(e[k] for k, _ in sr_b200.StreamEvent._fields_) for e in evs)


def _check_batch(h, pcm, evs, seg, atap):
    """the stream results equal the batch calls on the same samples: atap, segments, and segment 0's recognition"""
    want_a = h.noise_atap(pcm, 2400)
    want_s = h.vad(pcm, want_a)
    assert atap.tobytes() == want_a.tobytes() and np.array_equal(seg, want_s)
    closed = [(s, k) for s in range(len(pcm)) for k in range(3) if want_s[s, k, 1] != ob.NULL]
    assert sorted((e["stream"], e["segment"]) for e in evs) == closed and closed
    want = h.recognise(pcm, 2400, want=("best_idx", "best_dis", "cmd", "status"))
    for e in evs:
        if e["segment"] == 0:
            s = e["stream"]
            assert (e["best_idx"], e["best_dis"], e["cmd"], e["status"]) == tuple(int(want[q][s]) for q in ("best_idx", "best_dis", "cmd", "status"))


def _ragged_run(pool, pcm, rng, poison):
    S, L = pcm.shape
    pos, evs, k = np.zeros(S, np.int64), [], 0
    while (pos < L).any():
        lens = np.minimum(rng.choice([0, 0, 1, 81, 333, 1601, 4000], S), L - pos)
        lens[::5] = np.minimum(4000, L - pos[::5])                  # long rows next to empty ones
        if k % 2 == 0:
            lens[1::5] = 0
        k += 1
        w = int(lens.max()) + 24
        chunk = np.resize(np.asarray(poison, np.uint16), S * w).reshape(S, w)
        for s in range(S):
            chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
        evs += pool.push_ragged(chunk, lens)
        pos += lens
    return evs


@pytest.mark.parametrize("group", [False, True], ids=["pool", "group"])
def test_stream_push_reads_only_lens_samples(bank, group):
    """ragged pushes whose rows carry poison past lens[s] (lens 0 next to long rows), on one pool and on a stream group
    over the visible GPUs (two handles on one GPU without a second): the same events as clean pushes, equal to the batch"""
    import torch
    S, L = 25, 16000
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDA000, 2)
    ng = torch.cuda.device_count()
    hs = [_handle(bank) for _ in range(2)] if group and ng < 2 else [sr_b200.Handle(d) for d in range(ng)] if group else [_handle(bank)]
    for h in hs:
        h.set_bank(bank, T, 4096)
    runs = []
    for poison in ([0, 0], [0xFFFF, 0]):
        pool = sr_b200.StreamPool(hs if group else hs[0], S, L, 2400)
        evs = _ragged_run(pool, pcm, np.random.default_rng(4), poison)
        seg, atap = pool.segments()
        pool.close()
        runs.append((_events_key(evs), seg, atap))
        if poison[0] == 0xFFFF:
            _check_batch(hs[0], pcm, evs, seg, atap)
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1]) and runs[0][2].tobytes() == runs[1][2].tobytes()
    for h in hs:
        h.close()


def test_stream_lock_step_reads_only_chunk_len_from_pinned_strided_rows(bank):
    """lock-step pushes from pinned host memory, rows chunk_stride > chunk_len apart with poison in between"""
    S, L, cl, stride = 24, 16000, 800, 808 + 13
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDB000, 2)
    h = _handle(bank)
    buf, p = sr_b200.host_alloc_dev(0, S * stride * 2)
    try:
        rows = buf.view(np.uint16).reshape(S, stride)
        pool = sr_b200.StreamPool(h, S, L, 2400)
        evs = []
        for n0 in range(0, L, cl):
            rows[:] = np.resize(np.array([0xFFFF, 0], np.uint16), stride)
            rows[:, :cl] = pcm[:, n0:n0 + cl]
            evs += pool.push(p, chunk_len=cl, stride=stride)
        seg, atap = pool.segments()
        pool.close()
    finally:
        sr_b200.host_free(p)
    _check_batch(h, pcm, evs, seg, atap)
    h.close()


@pytest.mark.parametrize("ragged", [False, True], ids=["lock_step", "ragged"])
def test_stream_push_past_max_samples_drops_the_excess(bank, ragged):
    """16 000 samples pushed into 12 000-sample streams, lock-step or ragged (some pushes straddle the end): the excess
    is dropped, events and sr_streams_segments equal the batch results on the first 12 000 samples"""
    S, L, N = 20, 12000, 16000
    pcm = sr_b200.synth_pcm_host(S, N, 0x5EEDC000, 2)
    pcm[:, L:] = np.resize(np.array([4095, 0], np.uint16), N - L)   # loud: a segment would open if they were appended
    h = _handle(bank)
    pool = sr_b200.StreamPool(h, S, L, 2400)
    evs = []
    if ragged:
        rng = np.random.default_rng(12)
        pos = np.zeros(S, np.int64)
        while (pos < N).any():
            lens = np.minimum(rng.choice([0, 700, 1000, 2500], S), N - pos)
            w = max(int(lens.max()), 1)
            chunk = np.zeros((S, w), np.uint16)
            for s in range(S):
                chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
            evs += pool.push_ragged(chunk, lens)
            pos += lens
    else:
        for n0 in range(0, N, 1000):
            evs += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 1000]))
    seg, atap = pool.segments()
    pool.close()
    _check_batch(h, np.ascontiguousarray(pcm[:, :L]), evs, seg, atap)
    h.close()


# ---- one grammar decode per long recording (include/sr_long_grammar.h) ------------------------------------------------------
G13 = (3, 5, [(0, 1, 0x3), (1, 2, 0x7), (2, 0, 0x7), (1, 1, 0x8)])    # 3 states over commands 0-3


def _long_gram_oracle(pcm, n_len, bank_, n_slot, stride, g, P, max_segs, max_words, lens=None, geom_b=False, atap=None):
    return ox.recognise_long_grammar(ox.long_oracle(), ob.port(), ox.long_grammar(), pcm, n_len, bank_, n_slot, stride, g,
                                     P, max_segs, max_words, lens, geom_b, atap)


def _same(got, want, what=""):
    for k in want:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), (what, k)


@pytest.mark.parametrize("geom", [0, 1], ids=["ref", "geom_b"])
def test_long_grammar_reads_only_lens_samples(bank, geom):
    """sr_recognise_long_grammar_batch: loud band-crossing poison past lens[b] (it would open segments if read) gives the
    results of the clean recordings, which equal the composed oracle"""
    B, U = 5, 90001
    lens = np.array([U, 70000, 2399, 161, 40000], np.uint32)
    clean = ox.synth_long(B, U, 0x13A5)
    bad = clean.copy()
    for b, n in enumerate(lens):
        bad[b, n:] = np.where(np.arange(U - n) % 2, 4095, 0)
    want = _long_gram_oracle(clean, 2400, bank, T, 4096, G13, 1000, 64, 256, lens, geom == 1)
    assert (want["n_segs"][[0, 1, 4]] >= 3).all() and (want["n_words"] > 0).sum() >= 3
    h = _handle(bank, geom)
    for pcm in (clean, bad):
        _same(h.recognise_long_grammar(pcm, G13, 1000, 64, 256, 2400, lens), want, "poison" if pcm is bad else "clean")
    h.close()


def test_long_grammar_outputs_may_be_null(bank):
    """each output pointer NULL in turn, and every one but n_words: the fields passed equal the full call's. With atap
    NULL and n_len = 0 (no calibration overwrites it) the call starts from zeros although the previous call on the handle
    left another atap in the workspace the NULL path uses"""
    B, U, MS, MW = 4, 60001, 5, 40
    lens = np.array([U, 2000, 50000, 30000], np.uint32)
    pcm = ox.synth_long(B, U, 0x13A6)
    h = _handle(bank)
    full = h.recognise_long_grammar(pcm, G13, 1000, MS, MW, 2400, lens)
    _same(full, _long_gram_oracle(pcm, 2400, bank, T, 4096, G13, 1000, MS, MW, lens))
    assert (full["n_segs"] > MS).any() and (full["n_words"] > 0).sum() >= 2
    F = sr_b200.LONG_GRAM_FIELDS
    for want in [tuple(k for k in F if k != q) for q in F] + [("n_words",)]:
        _same(h.recognise_long_grammar(pcm, G13, 1000, MS, MW, 2400, lens, want=want), {k: full[k] for k in want}, want)
    # n_len = 0: atap is the one VAD uses from the first sample on
    given = _front(pcm, U)
    assert (given["mid_val"] != 0).all()
    out = {k: np.zeros(full[k].shape, full[k].dtype) for k in F}
    out["atap"] = given.copy()
    with_given = h.recognise_long_grammar(pcm, G13, 1000, MS, MW, 0, lens, out=out)   # leaves `given` in the workspace
    assert with_given["atap"].tobytes() == given.tobytes()
    no_atap = tuple(k for k in F if k != "atap")
    got = h.recognise_long_grammar(pcm, G13, 1000, MS, MW, 0, lens, want=no_atap)
    want = _long_gram_oracle(pcm, 0, bank, T, 4096, G13, 1000, MS, MW, lens)
    _same(got, {k: want[k] for k in no_atap}, "atap NULL after a call with another atap")
    assert any(got[k].tobytes() != with_given[k].tobytes() for k in no_atap)      # stale bytes would show
    h.close()


def test_long_grammar_shares_workspaces_with_the_other_calls(ora):
    """on one handle: a 16-state K13 decode of a 2^27-sample recording (its records grow the workspace past 256 MB), a
    1-state sr_connected_grammar_segs_batch, a larger sr_recognise_long_batch, a small K13 call in each geometry, the
    capture grammar and connected calls, then K13 with a larger batch. Each result equals a fresh handle's byte for
    byte, and the fresh handle's equals the CPU oracles"""
    from test_connected import _bank
    from test_long_stream import plant_act, planted_atap
    lo, port = ox.long_oracle(), ob.port()
    bk = _bank(np.random.default_rng(0x13F1), 16, "small", plant=False)     # 16 slots of 1-8 frames, stride 2880
    NS, ST = 16, bk.shape[1]
    g16 = (16, 0xFFFF, [(k, (k + 1) % 16, 0x1) for k in range(16)])          # 16 states x the 4 slots of command 0
    chain = sr_b200.chain_grammar(3, 0xF)
    # 800 active frames, 11 inactive: segments of 800 frames, 98.6 % of the recording decodable
    act = ((np.arange((1 << 27) // 80 - 1) % 811) < 800).astype(np.uint8)
    big = np.ascontiguousarray(plant_act(act)[None, :1 << 27])
    assert act.sum() * 16 * 12 > 256 << 20
    rng = np.random.default_rng(0x13F2)
    seg_frm = np.array([7, 0, 300, 1, 818], np.uint32)
    feat = rng.integers(-3000, 3001, (int(seg_frm.sum()), 12)).astype(np.int16)
    seq_seg = np.array([0, 2, 5], np.uint32)
    pcm3 = ox.synth_long(12, 100000, 0x13F3)
    pcm4 = ox.synth_long(3, 30000, 0x13F4)
    pcm5 = sr_b200.synth_pcm_host(8, 16000, 0x13F5, 3)
    lens6 = np.array([60000, 59000, 20000, 161, 60000, 45000, 2401, 60000], np.uint32)
    pcm6 = ox.synth_long(8, 60000, 0x13F6)

    def steps():
        yield "big", lambda h: h.recognise_long_grammar(big, g16, 1000, 8, 32, 0, None,
                                                        out=dict(_gram_out(1, 8, 32), atap=planted_atap(1)))
        yield "segs", lambda h: dict(zip(("words", "n_words", "total"), h.connected_grammar_segs(feat, seq_seg, seg_frm,
                                                                                                 sr_b200.loop_grammar(), 500, 64)))
        yield "long_batch", lambda h: h.recognise_long_batch(pcm3, 96, 2400)
        for geom in (0, 1):
            yield "small_geom%d" % geom, lambda h, geom=geom: _in_geom(h, geom, lambda: h.recognise_long_grammar(pcm4, chain, 1000, 16, 16))
        yield "capture", lambda h: dict([("g_" + k, a) for k, a in h.recognise_connected_grammar(pcm5, chain, 0, 8).items()] +
                                        [("c_" + k, a) for k, a in h.recognise_connected(pcm5, 3000, 8).items()])
        yield "k13_larger_b", lambda h: h.recognise_long_grammar(pcm6, chain, 1000, 24, 64, 2400, lens6)

    def oracle(name, got):
        if name == "big":
            w = _long_gram_oracle(big, 0, bk, NS, ST, g16, 1000, 8, 32, atap=planted_atap(1))
            assert int(w["n_segs"][0]) > 2000 and int(w["n_words"][0]) > 2000
        elif name == "segs":
            w = dict(zip(("words", "n_words", "total"), ox.long_grammar().decode_segs(feat, seq_seg, seg_frm, bk, NS, ST,
                                                                                       sr_b200.loop_grammar(), 500, 64)))
        elif name == "long_batch":
            w = ox.recognise_long(lo, port, pcm3, 2400, bk, NS, ST, 96)
        elif name.startswith("small"):
            w = _long_gram_oracle(pcm4, 2400, bk, NS, ST, chain, 1000, 16, 16, geom_b=name.endswith("1"))
        elif name == "capture":
            a = ox.recognise_connected_grammar(ora, ox.grammar(), pcm5, 2400, bk, NS, ST, chain, 0, 8)
            b = ox.recognise_connected(ora, ox.connected(), pcm5, 2400, bk, NS, ST, 3000, 8)
            w = dict([("g_" + k, v) for k, v in a.items()] + [("c_" + k, v) for k, v in b.items()])
        else:
            w = _long_gram_oracle(pcm6, 2400, bk, NS, ST, chain, 1000, 24, 64, lens6)
        _same(got, w, name + " (fresh handle) against the oracle")

    shared = _handle()
    shared.set_bank(bk, NS, ST)
    try:
        for name, run in steps():
            got = run(shared)
            fresh = _handle()
            fresh.set_bank(bk, NS, ST)
            want = run(fresh)
            fresh.close()
            _same(got, want, name + ": shared handle against a fresh one")
            oracle(name, want)
    finally:
        shared.close()


def _gram_out(B, max_segs, max_words):
    shape = {"atap": (B, ob.ATAP_DTYPE), "n_segs": (B, np.uint32), "seg_off": ((B, max_segs, 2), np.uint32),
             "frm_num": ((B, max_segs), np.uint32), "seg_status": ((B, max_segs), np.uint8), "n_words": (B, np.uint32),
             "words": ((B, max_words), sr_b200.WORD_DTYPE), "total": (B, np.uint64)}
    return {k: np.zeros(*shape[k]) for k in sr_b200.LONG_GRAM_FIELDS}


def _in_geom(h, geom, f):
    h.set_geometry(geom)
    try:
        return f()
    finally:
        h.set_geometry(0)


# ---- live streams of any length (include/sr_long_stream.h) ---------------------------------------------------------------
def _long_events(evs, S):
    """each stream's event records in segment order"""
    per = [[] for _ in range(S)]
    for e in sorted(evs, key=lambda e: (e["stream"], e["segment"])):
        assert e["segment"] == len(per[e["stream"]])
        per[e["stream"]].append(tuple(int(e[k]) for k in ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")))
    return per


def _check_long_prefix(h, pcm, per, st, n_len=2400):
    """prefix equality after the last push: each stream's events are the closed records of sr_recognise_long_batch on
    what it was fed, open_start its open record, atap its atap"""
    S, N = pcm.shape
    r = h.recognise_long_batch(pcm, N // 1520 + 4, n_len)
    for s in range(S):
        recs = [tuple(int(v) for v in rec) for rec in r["segs"][s, :int(r["n_segs"][s])].tolist()]
        assert per[s] == [t for t in recs if t[2] != 1], s
        assert int(st["open_start"][s]) == (recs[-1][0] if recs and recs[-1][2] == 1 else ob.NULL), s
        assert st["atap"][s].tobytes() == r["atap"][s].tobytes() and int(st["n_recv"][s]) == N
    assert sum(len(p) for p in per) > S


def test_long_stream_push_reads_only_lens_samples(bank):
    """sr_long_streams_push_ragged with rows that carry poison past lens[s] (lens 0 next to long rows): the events and
    state of clean pushes, which satisfy prefix equality"""
    S, L = 25, 40000
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDD000, 2)
    h = _handle(bank)
    runs = []
    for poison in ([0, 0], [0xFFFF, 0]):
        pool = sr_b200.LongStreamPool(h, S, 4000, 2400)
        evs = _ragged_run(pool, pcm, np.random.default_rng(14), poison)
        st = pool.state()
        pool.close()
        runs.append((_long_events(evs, S), st))
    assert runs[0][0] == runs[1][0] and all(runs[0][1][k].tobytes() == runs[1][1][k].tobytes() for k in runs[0][1])
    _check_long_prefix(h, pcm, runs[1][0], runs[1][1])
    h.close()


def test_long_stream_lock_step_reads_only_chunk_len_from_pinned_strided_rows(bank):
    """sr_long_streams_push from pinned host memory, rows chunk_stride > chunk_len apart with poison in between: the
    events and state of pushes of clean rows"""
    S, L, cl, stride = 24, 16000, 800, 808 + 13
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDE000, 2)
    h = _handle(bank)
    buf, p = sr_b200.host_alloc_dev(0, S * stride * 2)
    runs = []
    try:
        rows = buf.view(np.uint16).reshape(S, stride)
        for pinned in (False, True):
            pool = sr_b200.LongStreamPool(h, S, cl, 2400)
            evs = []
            for n0 in range(0, L, cl):
                if pinned:
                    rows[:] = np.resize(np.array([0xFFFF, 0], np.uint16), stride)
                    rows[:, :cl] = pcm[:, n0:n0 + cl]
                    evs += pool.push(p, chunk_len=cl, stride=stride)
                else:
                    evs += pool.push(np.ascontiguousarray(pcm[:, n0:n0 + cl]))
            runs.append((_long_events(evs, S), pool.state()))
            pool.close()
    finally:
        sr_b200.host_free(p)
    assert runs[0][0] == runs[1][0] and all(runs[0][1][k].tobytes() == runs[1][1][k].tobytes() for k in runs[0][1])
    _check_long_prefix(h, pcm, runs[1][0], runs[1][1])
    h.close()


def test_long_stream_reset_leaves_no_stale_ring_content(bank):
    """rings and mirrors filled with MARK / LOUD blocks, then a subset reset and planted audio pushed to the reset streams:
    a segment at stream sample 0, one on ring slot 0 after the first wrap (x[-1] from the mirror's partner slot R - 1)
    and one across the wrap, read through the mirror. Events and state() equal a fresh pool's"""
    from test_long_stream import MARK, plant_segs, planted_atap
    h = _handle(bank)
    h.set_bank(bank, T, 4096)
    S, mc = 6, 640
    which = (np.arange(S) % 2 == 0).astype(np.uint8)
    pool = sr_b200.LongStreamPool(h, S, mc, 0, planted_atap(S))
    Rb = pool.ring_len // 80
    x = plant_segs(4 * Rb, [(0, 30), (Rb, 40), (2 * Rb - 20, 60)])
    stale = np.tile(np.repeat(np.array([MARK, 2148], np.uint16), 80), Rb + 200)[:2 * 80 * Rb + 777]
    try:
        for n0 in range(0, len(stale), mc):
            pool.push(np.ascontiguousarray(np.tile(stale[n0:n0 + mc], (S, 1))))
        kept = pool.state()
        pool.reset(which, planted_atap(S))
        fresh = sr_b200.LongStreamPool(h, S, mc, 0, planted_atap(S))
        got, want = [], []
        for n0 in range(0, len(x), mc):
            k = min(mc, len(x) - n0)
            chunk = np.zeros((S, k), np.uint16)
            chunk[which == 1] = x[n0:n0 + k]
            lens = np.where(which == 1, k, 0).astype(np.uint32)
            got += pool.push_ragged(chunk, lens)
            want += fresh.push_ragged(chunk, lens)
        st, fs = pool.state(), fresh.state()
        fresh.close()
        r = which == 1
        assert _long_events(got, S) == _long_events(want, S)
        assert [len(p) for p in _long_events(got, S)] == [3 if w else 0 for w in which]
        for k in st:
            assert st[k][r].tobytes() == fs[k][r].tobytes(), k
            assert st[k][~r].tobytes() == kept[k][~r].tobytes(), k
    finally:
        pool.close()
    h.close()


def test_long_stream_reset_drops_only_the_reset_streams_queued_events(bank):
    """events queued for reset and kept streams at the reset: each kept stream's survive in order, the reset streams' are
    gone. Compared per stream with the same pool without the reset: within one push the order across streams is that of
    the step kernel's atomic event slots, so only each stream's own sequence is defined"""
    S, L, mc = 6, 48000, 640
    pcm = sr_b200.synth_pcm_host(S, L, 0x5EEDF000, 3)
    h = _handle(bank)
    which = np.array([1, 0, 0, 1, 0, 1], np.uint8)
    out = []
    for reset in (False, True):
        pool = sr_b200.LongStreamPool(h, S, mc, 2400)
        for n0 in range(0, L, mc):
            assert pool.push(np.ascontiguousarray(pcm[:, n0:n0 + mc]), max_events=0) == []
        queued = pool.pending()
        if reset:
            pool.reset(which)
        out.append((queued, pool.fetch(max_events=max(queued, 1)), pool.pending()))
        pool.close()
    (q0, all_ev, p0), (q1, kept_ev, p1) = out
    assert q0 == q1 and p0 == p1 == 0

    def per_stream(evs):                                            # each stream's events in the order handed out
        return [[e for e in evs if e["stream"] == s] for s in range(S)]
    every, kept = per_stream(all_ev), per_stream(kept_ev)
    assert all(every[s] for s in range(S))
    for s in range(S):
        if which[s]:
            assert kept[s] == [], s
        else:
            assert kept[s] == every[s] and [e["segment"] for e in kept[s]] == list(range(len(kept[s]))), s
    h.close()


def test_long_stream_state_outputs_may_be_null(bank):
    """sr_long_streams_state with each output NULL in turn equals the full query, and leaves the caller's arrays it was
    not given alone"""
    S = 9
    pcm = sr_b200.synth_pcm_host(S, 24000, 0x5EEE0000, 3)
    h = _handle(bank)
    pool = sr_b200.LongStreamPool(h, S, 800, 2400)
    try:
        for n0 in range(0, 24000 - 333, 800):
            pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 800]))
        full = pool.state()
        assert (full["n_closed"] > 0).any() and (full["n_recv"] > 0).all()
        keys = ("n_recv", "n_closed", "open_start", "atap")
        for null in keys + (None,):
            arr = {k: np.frombuffer(b"\xa5" * full[k].nbytes, full[k].dtype).copy() for k in keys}
            assert sr_b200.lib().sr_long_streams_state(pool._p, *[None if k == null else arr[k].ctypes.data for k in keys]) == 0
            for k in keys:
                if k == null:
                    assert set(arr[k].tobytes()) == {0xA5}, k
                else:
                    assert arr[k].tobytes() == full[k].tobytes(), (null, k)
    finally:
        pool.close()
    h.close()
