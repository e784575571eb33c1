"""ctypes bindings of the two checkers (TEST INFRASTRUCTURE):
  oracle/_build/liboracle.so  -- our C restatement (sr_oracle.c), re-entrant, multi-threaded batches
  oracle/_ref/libref.so       -- the reference's own VAD.C/MFCC.C/DTW.C compiled for the host (non re-entrant)
Both expose the same Python surface so tests can run against either."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PORT_SO = os.path.join(ROOT, "oracle", "_build", "liboracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref.so")

ATAP_DTYPE = np.dtype([("mid_val", "<u4"), ("n_thl", "<u2"), ("z_thl", "<u2"), ("s_thl", "<u4")])
FTR_DTYPE = np.dtype([("save_sign", "<u2"), ("frm_num", "<u2"), ("mfcc_dat", "<i2", (119 * 12,))])
NULL = 0xFFFFFFFF


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ftr_rows(ftr):
    """list of (frm_num, rows[frm_num,12]) -- only the part get_mfcc defines"""
    out = []
    for i in range(ftr.shape[0]):
        n = int(ftr["frm_num"][i])
        out.append((n, ftr["mfcc_dat"][i][: n * 12].copy()))
    return out


def ftr_equal(a, b):
    if not np.array_equal(a["frm_num"], b["frm_num"]):
        return False
    n = a["frm_num"].astype(np.int64) * 12
    mask = np.arange(119 * 12)[None, :] < n[:, None]
    return bool(np.array_equal(np.where(mask, a["mfcc_dat"], 0), np.where(mask, b["mfcc_dat"], 0)))


class _Base:
    name = "?"

    def recognise_batch(self, pcm, n_len, bank, n_slot, slot_stride, nthreads=1):
        raise NotImplementedError


class PortOracle(_Base):
    name = "oracle-port"

    def __init__(self):
        self.lib = C.CDLL(PORT_SO)
        self.lib.sro_dtw.restype = C.c_uint32
        self.lib.sro_dtw_band.restype = C.c_uint32
        self.lib.sro_get_dis.restype = C.c_uint32
        self.lib.sro_log100.restype = C.c_uint32
        self.lib.sro_log100.argtypes = [C.c_uint32]
        self.lib.sro_dtw_limit.argtypes = [C.c_int] * 4

    def noise_atap(self, pcm1d, n_len, atap=None):
        a = np.zeros(1, ATAP_DTYPE) if atap is None else atap.copy().reshape(1)
        self.lib.sro_noise_atap(_p(pcm1d), C.c_uint32(n_len), _p(a))
        return a

    def vad(self, pcm1d, buf_len, atap):
        seg = np.zeros(6, np.uint32)
        self.lib.sro_vad(_p(pcm1d), C.c_uint32(buf_len), _p(atap), _p(seg))
        return seg

    def fft_raw(self, packed):
        out = np.zeros_like(packed)
        for i in range(packed.shape[0]):
            self.lib.sro_fft_raw(_p(packed[i]), _p(out[i]))
        return out

    def fft_mag(self, frames):
        n, ln = frames.shape
        out = np.zeros((n, 512), np.uint32)
        for i in range(n):
            self.lib.sro_fft_mag(_p(frames[i]), C.c_uint32(ln), _p(out[i]))
        return out

    def mfcc_batch(self, pcm, seg2, atap, nthreads=1):
        B, U = pcm.shape
        ftr = np.zeros(B, FTR_DTYPE)
        seg2 = np.ascontiguousarray(seg2, np.uint32).reshape(B, 2)
        self.lib.sro_mfcc_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), _p(seg2), _p(atap), _p(ftr), C.c_int(nthreads))
        return ftr

    def mfcc_geom_b_batch(self, pcm, seg2, atap):
        """GEOM_B extension (200/80/256): this repo's own restatement is its only checker (parity unpinned)"""
        B, U = pcm.shape
        ftr = np.zeros(B, FTR_DTYPE)
        seg2 = np.ascontiguousarray(seg2, np.uint32).reshape(B, 2)
        self.lib.sro_mfcc_geom_b_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), _p(seg2), _p(atap), _p(ftr))
        return ftr

    def fft_raw_n(self, packed, N):
        out = np.zeros_like(packed)
        for i in range(packed.shape[0]):
            self.lib.sro_fft_raw_n(_p(packed[i]), _p(out[i]), C.c_uint32(N))
        return out

    def get_dis(self, a, b):
        return np.array([self.lib.sro_get_dis(_p(a[i]), _p(b[i])) for i in range(a.shape[0])], np.uint32)

    def get_mdl(self, f1, f2):
        self.lib.sro_get_mdl.restype = C.c_uint32
        n = f1.shape[0]
        mdl, dis = np.zeros(n, FTR_DTYPE), np.zeros(n, np.uint32)
        for i in range(n):
            dis[i] = self.lib.sro_get_mdl(_p(f1[i:i + 1]), _p(f2[i:i + 1]), _p(mdl[i:i + 1]))
        return mdl, dis

    def dtw_batch(self, ftr_in, bank, n_slot, slot_stride, check_sign=0, band_r=-1, nthreads=1):
        B = ftr_in.shape[0]
        score = np.zeros((B, n_slot), np.uint32)
        cells = C.c_uint64(0)
        self.lib.sro_dtw_batch(_p(ftr_in), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
                               C.c_int(check_sign), C.c_int(band_r), _p(score), C.byref(cells), C.c_int(nthreads))
        return score, int(cells.value)

    def recognise_batch(self, pcm, n_len, bank, n_slot, slot_stride, nthreads=1):
        B, U = pcm.shape
        out = dict(atap=np.zeros(B, ATAP_DTYPE), seg_off=np.zeros((B, 3, 2), np.uint32), ftr=np.zeros(B, FTR_DTYPE),
                   score=np.zeros((B, n_slot), np.uint32), best_idx=np.zeros(B, np.uint32),
                   best_dis=np.zeros(B, np.uint32), cmd=np.zeros(B, np.uint32), status=np.zeros(B, np.uint8))
        if n_slot == 0:
            bank = np.zeros(16, np.uint8)
        self.lib.sro_recognise_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), C.c_uint32(n_len), _p(bank),
                                     C.c_uint32(n_slot), C.c_uint32(slot_stride), _p(out["atap"]), _p(out["seg_off"]),
                                     _p(out["ftr"]), _p(out["score"]), _p(out["best_idx"]), _p(out["best_dis"]),
                                     _p(out["cmd"]), _p(out["status"]), C.c_int(nthreads))
        # the reference never reaches dtw when VAD/MFCC fail: scores stay undefined -> pin to DIS_ERR for comparison
        out["score"][out["status"] != 0] = NULL
        return out


class RefOracle(_Base):
    """The reference's own C (unmodified VAD.C / MFCC.C / DTW.C) through oracle/ref_driver.c."""
    name = "reference-C"

    def __init__(self):
        self.lib = C.CDLL(REF_SO)
        self.lib.dtw.restype = C.c_uint32
        self.lib.get_dis.restype = C.c_uint32
        self.lib.dtw_limit.restype = C.c_uint8

    def noise_atap(self, pcm1d, n_len, atap=None):
        a = np.zeros(1, ATAP_DTYPE) if atap is None else atap.copy().reshape(1)
        self.lib.noise_atap(_p(pcm1d), C.c_uint16(n_len), _p(a))
        return a

    def vad(self, pcm1d, buf_len, atap):
        # ref_vad runs noise_atap first; call VAD alone through a zero-length noise window (n_len=1 is rejected -> untouched)
        seg = np.zeros(6, np.uint32)
        a = atap.copy().reshape(1)
        self.lib.ref_vad(_p(pcm1d), C.c_uint32(buf_len), C.c_uint32(1), _p(a), _p(seg))
        return seg

    def fft_raw(self, packed):
        out = np.zeros_like(packed)
        for i in range(packed.shape[0]):
            self.lib.ref_fft_raw(_p(packed[i]), _p(out[i]))
        return out

    def fft_mag(self, frames):
        n, ln = frames.shape
        out = np.zeros((n, 512), np.uint32)
        for i in range(n):
            self.lib.ref_fft_mag(_p(frames[i]), C.c_uint32(ln), _p(out[i]))
        return out

    def mfcc_batch(self, pcm, seg2, atap, nthreads=1):
        B, U = pcm.shape
        ftr = np.zeros(B, FTR_DTYPE)
        seg2 = np.ascontiguousarray(seg2, np.uint32).reshape(B, 2)
        self.lib.ref_mfcc_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), _p(seg2), _p(atap), _p(ftr))
        return ftr

    def get_dis(self, a, b):
        return np.array([self.lib.get_dis(_p(a[i]), _p(b[i])) for i in range(a.shape[0])], np.uint32)

    def get_mdl(self, f1, f2):
        """the reference's own get_mdl (DTW.C:217); only safe for paths of <= 119 points (it does not bound its writes)"""
        self.lib.get_mdl.restype = C.c_uint32
        n = f1.shape[0]
        mdl, dis = np.zeros(n, FTR_DTYPE), np.zeros(n, np.uint32)
        for i in range(n):
            dis[i] = self.lib.get_mdl(_p(f1[i:i + 1]), _p(f2[i:i + 1]), _p(mdl[i:i + 1]))
        return mdl, dis

    def dtw_batch(self, ftr_in, bank, n_slot, slot_stride, check_sign=0, band_r=-1, nthreads=1):
        assert band_r < 0, "the reference has no banded DP"
        B = ftr_in.shape[0]
        score = np.zeros((B, n_slot), np.uint32)
        self.lib.ref_dtw_batch(_p(ftr_in), C.c_uint32(B), _p(bank), C.c_uint32(n_slot), C.c_uint32(slot_stride),
                               C.c_int(check_sign), _p(score))
        return score, None

    def recognise_batch(self, pcm, n_len, bank, n_slot, slot_stride, nthreads=1):
        B, U = pcm.shape
        out = dict(seg_off=np.zeros((B, 3, 2), np.uint32), ftr=np.zeros(B, FTR_DTYPE),
                   score=np.zeros((B, n_slot), np.uint32), best_idx=np.zeros(B, np.uint32),
                   best_dis=np.zeros(B, np.uint32), cmd=np.zeros(B, np.uint32), status=np.zeros(B, np.uint8))
        if n_slot == 0:
            bank = np.zeros(16, np.uint8)
        self.lib.ref_recognise_batch(_p(pcm), C.c_uint32(U), C.c_uint32(B), C.c_uint32(n_len), _p(bank),
                                     C.c_uint32(n_slot), C.c_uint32(slot_stride), _p(out["seg_off"]), _p(out["ftr"]),
                                     _p(out["score"]), _p(out["best_idx"]), _p(out["best_dis"]), _p(out["cmd"]),
                                     _p(out["status"]))
        out["score"][out["status"] != 0] = NULL
        # a failed VAD leaves ftr untouched in the reference; the batched API reports frm_num = 0
        return out


def pinned_rows(pcm, atap):
    """rows of U + 1 samples, [mid_val, row...]: with every segment shifted by +1, x[-1] of a segment that starts at
    sample 0 is the utterance's own mid_val (as a 16-bit sample), and every other segment reads its own samples"""
    B, U = pcm.shape
    rows = np.empty((B, U + 1), np.uint16)
    rows[:, 0] = atap["mid_val"].astype(np.uint16)
    rows[:, 1:] = pcm
    return rows


def plant_sample0(pcm, rows, seed, before=4095):
    """make VAD open segment 0 of each of `rows` at sample 0 (in place): someone is already speaking when the capture
    starts. The first 560..1400 samples alternate between m +- 1200 (+- 150 of noise), m = the level of the quiet that
    follows. The burst lies inside the 2 400-sample noise window, whose n_thl is the MEAN of the per-240-sample maxima
    (VAD.C:60-68): at most 6 of its 10 windows are loud, so n_thl stays below 900 and every sample of the burst crosses
    the band (frm_zero > z_thl); frames 0-7 are active and the segment is back-dated to sample 0 (VAD.C:178). The quiet
    after the burst closes it: 8..18 frames. The last sample of the row before each planted row is set to `before`, far
    from m, so x[-1] read from the neighbour would change the features."""
    rng = np.random.default_rng(seed)
    for r in rows:
        n = int(rng.integers(640, 1400))
        m = int(round(float(pcm[r, 1400:2400].mean())))
        burst = m + np.where(np.arange(n) % 2 == 0, 1200, -1200) + rng.integers(-150, 151, n)
        pcm[r, :n] = np.clip(burst, 0, 4095)
        if r > 0:
            pcm[r - 1, -1] = before


def recognise_pinned(ora, pcm, n_len, bank, n_slot, slot_stride, geom_b=False):
    """recognise_batch composed from the oracle's own stages, one utterance at a time, with x[-1] of a segment that starts
    at sample 0 pinned to that utterance's mid_val (the rule of every batched entry point): noise_atap and VAD on the row,
    get_mfcc of segment 0 on pinned_rows, dtw with the save_sign check, the strict '<' first-wins argmin (main.c:276-294).
    geom_b: the GEOM_B get_mfcc (the port's restatement only). Same dict as recognise_batch."""
    B, U = pcm.shape
    out = dict(atap=np.zeros(B, ATAP_DTYPE), seg_off=np.zeros((B, 3, 2), np.uint32), ftr=np.zeros(B, FTR_DTYPE),
               score=np.full((B, n_slot), NULL, np.uint32), best_idx=np.zeros(B, np.uint32),
               best_dis=np.full(B, NULL, np.uint32), cmd=np.zeros(B, np.uint32), status=np.ones(B, np.uint8))
    for b in range(B):
        out["atap"][b] = ora.noise_atap(pcm[b], n_len)[0]
        out["seg_off"][b] = ora.vad(pcm[b], U, out["atap"][b:b + 1]).reshape(3, 2)
    ok = out["seg_off"][:, 0, 1] != NULL                      # main.c:261-266: VAD found no segment -> status 1
    if ok.any():
        rows = pinned_rows(pcm[ok], out["atap"][ok])
        seg = out["seg_off"][ok, 0, :] + 1
        f = ora.mfcc_geom_b_batch(rows, seg, out["atap"][ok]) if geom_b else ora.mfcc_batch(rows, seg, out["atap"][ok])
        out["ftr"][ok] = f
    out["status"][ok] = np.where(out["ftr"]["frm_num"][ok] == 0, 2, 0)   # main.c:269-274
    good = out["status"] == 0
    if good.any() and n_slot:
        sc, _ = ora.dtw_batch(out["ftr"][good], bank, n_slot, slot_stride, check_sign=1)
        out["score"][good] = sc
        i = np.argmin(sc, axis=1)                             # first of the minima == the strict '<' scan from DIS_ERR
        out["best_idx"][good] = i
        out["best_dis"][good] = sc[np.arange(sc.shape[0]), i]
        out["cmd"][good] = i // 4
    return out


def have_ref():
    return os.path.exists(REF_SO)


def port():
    return PortOracle()


def ref():
    return RefOracle()


def best_oracle():
    """The reference's own C when its prebuilt .so travelled with the repo, else our restatement."""
    return RefOracle() if have_ref() else PortOracle()
