"""Handles that share one GPU stay independent (include/speech_recog.h: "use one handle per thread ... Different handles --
on the same or on different GPUs -- are independent"; concurrent streams take one handle each; the drop-ins' dtw_limit
state, fft buffer and last error belong to the calling thread).

Every output of the library is integer and deterministic, so cross-talk between handles shows up as a bit difference
against a run made alone. The job table below runs one fixed script per entry-point family on a handle of its own; a
serial baseline runs each job alone (checked on a sample against its oracle), then every job runs R times at once, one
thread per handle. ctypes releases the GIL during each C call, so the threads' library calls overlap. Each job alternates
between two inputs, so a repetition that skips work and leaves the previous repetition's workspace contents behind
cannot pass. The last test is a CPU test: every sr_* entry point of every header under include/ (found by glob, so a new
header cannot stay out) is either in the job table or excluded with a reason."""
import ctypes as C
import glob
import os
import re
import subprocess
import sys
import threading
import time
import traceback

import numpy as np
import pytest

import oracle_bind as ob
import oracle_ext as ox
import sr_b200

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# every public header (include/compat/ holds the reference's own headers, which glob does not enter); sr_synth.h declares
# the synthetic-workload helpers the tests build inputs with, whose names may be listed but need no job
SYNTH_HEADER = os.path.join(ROOT, "include", "sr_synth.h")
HEADERS = tuple(sorted(h for h in glob.glob(os.path.join(ROOT, "include", "*.h")) if h != SYNTH_HEADER))

R = 3                                    # repetitions of every job in the concurrent run
TIMING_CAP = 512                         # timing records per handle: more than any job launches per repetition
VAD_, MFCC_, STATUS, BEST_INIT, DTW, BEST_FINAL, DTW_BAND, ALIGN, AVG_UPDATE, CONN, GRAM = range(11)
EVENT_DTYPE = np.dtype([(k, "<u4") for k, _ in sr_b200.StreamEvent._fields_])


# ---- comparison ---------------------------------------------------------------------------------------------------------
def first_diff(a, b):
    """None when a and b hold the same bytes, else where they first differ (element index, or shape / dtype)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return "shape/dtype %s %s vs %s %s" % (a.shape, a.dtype, b.shape, b.dtype)
    x, y = a.view(np.uint8).reshape(-1), b.view(np.uint8).reshape(-1)
    bad = np.nonzero(x != y)[0]
    if not len(bad):
        return None
    i = int(bad[0]) // max(a.itemsize, 1)
    return "first differing element %s of %s (%d bytes differ)" % (np.unravel_index(i, a.shape) if a.ndim else (), a.shape,
                                                                    len(bad))


def diff_outputs(got, want):
    """[(field, where)] for every field of two output dicts that differs"""
    out = [(k, "missing") for k in want if k not in got] + [(k, "unexpected") for k in got if k not in want]
    for k in want:
        if k in got:
            d = first_diff(got[k], want[k])
            if d:
                out.append((k, d))
    return out


def oracle_diff(got, want):
    """diff_outputs against an oracle: of feature structs only frm_num and the rows get_mfcc defines count"""
    out = []
    for k in want:
        if k in got and want[k].dtype == sr_b200.FTR_DTYPE:
            bad = [i for i in range(len(want[k])) if not ob.ftr_equal(got[k][i:i + 1], want[k][i:i + 1])]
            if bad:
                out.append((k, "features of row %d differ" % bad[0]))
    return out + diff_outputs({k: a for k, a in got.items() if a.dtype != sr_b200.FTR_DTYPE},
                              {k: a for k, a in want.items() if a.dtype != sr_b200.FTR_DTYPE})


def events_array(events):
    """stream events as one array sorted by (stream, segment): the order within one push is not defined"""
    names = EVENT_DTYPE.names
    return np.array(sorted(tuple(int(e[k]) for k in names) for e in events), dtype=EVENT_DTYPE)


def _argmin_rows(score):
    """best_idx / best_dis of main.c:285-289 (strict '<' from DIS_ERR, first wins) for each row of a score matrix"""
    key = (score.astype(np.uint64) << np.uint64(32)) | np.arange(score.shape[1], dtype=np.uint64)[None, :]
    k = key.min(axis=1)
    return (k & np.uint64(0xFFFFFFFF)).astype(np.uint32), (k >> np.uint64(32)).astype(np.uint32)


def _cpus():
    cpus = len(os.sched_getaffinity(0))
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        cpus = cpus if q == "max" else min(cpus, -(-int(q) // int(per)))
    except (OSError, ValueError):
        pass
    return cpus


# ---- inputs shared by the jobs (host only; built once) ------------------------------------------------------------------
class World:
    def __init__(self):
        self.ora = ob.best_oracle()
        self.po = ob.port()
        gold = np.load(os.path.join(HERE, "golden", "golden.npz"))
        self.bank8 = np.ascontiguousarray(gold["synth/bank"])          # 8 enrolled templates, flash layout
        tpl = sr_b200.synth_pcm_host(8, 8000, 0xC0C0B000)
        e = ob.recognise_pinned(self.po, tpl, 2400, None, 0, 4096, geom_b=True)
        assert (e["status"] == 0).all()
        self.bank_b = sr_b200.make_bank(e["ftr"])                        # the same for GEOM_B
        rng = np.random.default_rng(0xC0C0)
        b200 = sr_b200.synth_ftr_host(200, 0xC0C1000, 30, 119, stride=4096)
        bad = rng.random(200) < 0.33
        b200[bad, 0:2] = 0xFF                                            # erased flash: save_sign != 12345
        b200[~bad, 0], b200[~bad, 1] = sr_b200.SAVE_MASK & 0xFF, sr_b200.SAVE_MASK >> 8
        b200[7] = b200[3]                                                # a duplicate: first wins
        self.bank200 = b200
        b128 = sr_b200.synth_ftr_host(128, 0xC0C2000, 20, 80, stride=4096)
        b128[:, 0], b128[:, 1] = sr_b200.SAVE_MASK & 0xFF, sr_b200.SAVE_MASK >> 8
        self.bank128 = b128                                              # 128 members: 16-CTA decoder clusters
        words = sr_b200.synth_pcm_host(10, 8000, 0xC0C3000)
        e = ob.recognise_pinned(self.ora, words, 2400, None, 0, 4096)
        bank40 = np.full((40, 4096), 0xFF, np.uint8)
        bank40[::4] = sr_b200.make_bank(e["ftr"])
        bank40[::4][e["status"] != 0] = 0xFF
        self.bank40 = bank40                                             # one word per command at slot 4 * cmd, ten digits
        self._cache = {}

    def pcm(self, B, U, seed, nwords=1):
        k = (B, U, seed, nwords)
        if k not in self._cache:
            self._cache[k] = sr_b200.synth_pcm_host(B, U, seed, nwords)
        return self._cache[k]


# ---- the job table ------------------------------------------------------------------------------------------------------
class Job:
    """one fixed script on handles of its own (device 0). run(v) runs input variant v (0 or 1) and returns its outputs as
    numpy arrays; oracle(v, out) checks a sample of them against a plain reference."""
    name = "?"
    calls = ()                            # the C-ABI entry points run() reaches

    def __init__(self, w):
        self.w = w
        self.hs = []
        self.open()

    def handle(self, geom=0):
        h = sr_b200.Handle(0)
        h.timing_enable(TIMING_CAP)
        if geom:
            h.set_geometry(geom)
        self.hs.append(h)
        return h

    def open(self):
        raise NotImplementedError

    def close(self):
        for h in self.hs:
            h.close()
        self.hs = []

    def run(self, v):
        raise NotImplementedError

    def oracle(self, v, out):
        raise NotImplementedError

    def varying_launches(self):
        """launches of the last run() whose number legitimately depends on timing (none, except the packed transport)"""
        return 0


class RecognisePacked(Job):
    """sr_recognise_batch on host PCM, packed transport forced: four 32 MB chunks through the handle's packer pool and
    copy stream"""
    name = "recognise_packed"
    calls = ("sr_recognise_batch", "sr_set_transport", "sr_transport_stats", "sr_set_bank")
    B, U = 3 * 2096 + 8, 8000
    rows = (0, 1, 2095, 2096, 4191, 4192, 6295)

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank8, 8, 4096)
        self.h.set_transport(1)
        self.stats = []

    def run(self, v):
        out = self.h.recognise(self.w.pcm(self.B, self.U, 0xC1000000 + v))
        self.stats.append(self.h.transport_stats())
        return out

    def varying_launches(self):
        return self.stats[-1][0]          # one untimed 12-bit expansion per chunk that crossed packed

    def oracle(self, v, out):
        rows = list(self.rows)
        pcm = np.ascontiguousarray(self.w.pcm(self.B, self.U, 0xC1000000 + v)[rows])
        want = ob.recognise_pinned(self.w.ora, pcm, 2400, self.w.bank8, 8, 4096)
        return oracle_diff({k: out[k][rows] for k in want}, want)


class RecogniseDevBand(Job):
    """sr_recognise_batch_dev on device PCM from sr_synth_pcm_dev, on a torch stream of the job's own, with the banded DP
    matcher at r = 10 and then r = 118; outputs prefilled before each call"""
    name = "recognise_dev_band"
    calls = ("sr_recognise_batch_dev", "sr_set_stream", "sr_set_match", "sr_get_match", "sr_sync", "sr_synth_pcm_dev")
    B, U, T = 2048, 8000, 8
    rows = (0, 1, 777, 2047)

    def open(self):
        import torch
        self.torch = torch
        self.h = self.handle()
        self.h.set_bank(self.w.bank8, self.T, 4096)
        self.st = torch.cuda.Stream(torch.device("cuda:0"))
        self.h.set_stream(self.st.cuda_stream)
        with torch.cuda.stream(self.st):
            self.pcm = [torch.empty((self.B, self.U), dtype=torch.int16, device="cuda:0") for _ in range(2)]
            for v in range(2):
                sr_b200.synth_pcm_dev(self.pcm[v].data_ptr(), self.B, self.U, 0xC2000000 + v, 1, self.st.cuda_stream)
            self.out = {k: torch.empty(self.B * n, dtype=torch.uint8, device="cuda:0") for k, n in
                        (("atap", 12), ("seg_off", 24), ("ftr", sr_b200.FTR_BYTES), ("score", 4 * self.T), ("best_idx", 4),
                         ("best_dis", 4), ("cmd", 4), ("status", 1))}
        self.st.synchronize()

    def _host(self):
        o = {k: t.cpu().numpy() for k, t in self.out.items()}
        B = self.B
        return {"atap": o["atap"].view(sr_b200.ATAP_DTYPE), "seg_off": o["seg_off"].view(np.uint32).reshape(B, 3, 2),
                "ftr": o["ftr"].view(sr_b200.FTR_DTYPE), "score": o["score"].view(np.uint32).reshape(B, self.T),
                "best_idx": o["best_idx"].view(np.uint32), "best_dis": o["best_dis"].view(np.uint32),
                "cmd": o["cmd"].view(np.uint32), "status": o["status"]}

    def run(self, v):
        res = {}
        with self.torch.cuda.stream(self.st):
            for r in (10, 118):
                self.h.set_match(sr_b200.DTW_BAND, r)
                assert self.h.match() == (sr_b200.DTW_BAND, r)
                for t in self.out.values():
                    t.fill_(0x5A)
                self.h.recognise_dev(self.pcm[v].data_ptr(), self.U, self.B, 2400,
                                     **{k: t.data_ptr() for k, t in self.out.items()})
                self.h.sync()
                res.update({"%s_r%d" % (k, r): a for k, a in self._host().items()})
        return res

    def oracle(self, v, out):
        rows = list(self.rows)
        pcm = np.ascontiguousarray(sr_b200.synth_pcm_host(self.B, self.U, 0xC2000000 + v)[rows])
        bad = []
        for r in (10, 118):
            want = ob.recognise_pinned(self.w.po, pcm, 2400, self.w.bank8, self.T, 4096)
            good = want["status"] == 0
            sc, _ = self.w.po.dtw_batch(want["ftr"][good], self.w.bank8, self.T, 4096, check_sign=1, band_r=r)
            want["score"][good] = sc
            bi, bd = _argmin_rows(sc)
            want["best_idx"][good], want["best_dis"][good], want["cmd"][good] = bi, bd, bi // 4
            bad += [("r%d %s" % (r, k), d) for k, d in oracle_diff({k: out["%s_r%d" % (k, r)][rows] for k in want}, want)]
        return bad


class DtwDynamic(Job):
    """sr_dtw_batch with the dynamic greedy kernel against a 200-slot bank (slot order active), save_sign honoured"""
    name = "dtw_dynamic"
    calls = ("sr_dtw_batch", "sr_set_dtw_variant", "sr_synth_ftr_host")
    B = 3000
    rows = (0, 1, 1499, 2999)

    def open(self):
        self.h = self.handle()
        self.h.set_dtw_variant(1)
        self.h.set_bank(self.w.bank200, 200, 4096)

    def fin(self, v):
        return sr_b200.synth_ftr_host(self.B, 0xC3000000 + v, 30, 119).view(sr_b200.FTR_DTYPE).reshape(-1)

    def run(self, v):
        score, bi, bd = self.h.dtw(self.fin(v), flags=sr_b200.DTW_CHECK_SIGN)
        return {"score": score, "best_idx": bi, "best_dis": bd}

    def oracle(self, v, out):
        rows = list(self.rows)
        sc, _ = self.w.ora.dtw_batch(np.ascontiguousarray(self.fin(v)[rows]), self.w.bank200, 200, 4096, check_sign=1)
        bi, bd = _argmin_rows(sc)
        return oracle_diff({k: out[k][rows] for k in ("score", "best_idx", "best_dis")},
                            {"score": sc, "best_idx": bi, "best_dis": bd})


class GeomB(Job):
    """sr_recognise_batch on a GEOM_B handle (200/80/256 framing)"""
    name = "geom_b"
    calls = ("sr_recognise_batch", "sr_set_geometry", "sr_get_geometry")
    B, U = 2048, 8000
    rows = (0, 1, 1000, 2047)

    def open(self):
        self.h = self.handle(geom=1)
        assert sr_b200.lib().sr_get_geometry(self.h._h) == 1
        self.h.set_transport(0)
        self.h.set_bank(self.w.bank_b, 8, 4096)

    def run(self, v):
        return self.h.recognise(self.w.pcm(self.B, self.U, 0xC4000000 + v))

    def oracle(self, v, out):
        rows = list(self.rows)
        pcm = np.ascontiguousarray(self.w.pcm(self.B, self.U, 0xC4000000 + v)[rows])
        want = ob.recognise_pinned(self.w.po, pcm, 2400, self.w.bank_b, 8, 4096, geom_b=True)
        return oracle_diff({k: out[k][rows] for k in want}, want)


class EnrolAverageAlign(Job):
    """sr_enrol_batch of 32 commands x 4 repetitions, sr_average_bank (K = 4, r = 118, 2 iterations), then sr_dtw_path_batch
    of every enrolled slot against its command's averaged template (32 times over)"""
    name = "enrol_average_path"
    calls = ("sr_enrol_batch", "sr_average_bank", "sr_dtw_path_batch")
    G, K = 32, 4

    def open(self):
        self.h = self.handle()

    def pcm(self, v):
        return self.w.pcm(self.G * self.K, 8000, 0xC5000000 + v)

    def run(self, v):
        bank, status = self.h.enrol(self.pcm(v), 2400)
        avg, score, anchor = self.h.average_bank(bank, 4096, self.K, 118, 2)
        a = np.ascontiguousarray(bank[:, :sr_b200.FTR_BYTES]).view(sr_b200.FTR_DTYPE).reshape(-1)
        b = np.ascontiguousarray(avg[::self.K, :sr_b200.FTR_BYTES]).view(sr_b200.FTR_DTYPE).reshape(-1)
        b = np.repeat(b, self.K)
        dis, path, plen = self.h.dtw_path(np.tile(a, 32), np.tile(b, 32), 118)
        return {"bank": bank, "status": status, "avg": avg, "score": score, "anchor": anchor, "dis": dis, "path": path,
                "path_len": plen}

    def oracle(self, v, out):
        rows = [0, 1, 2, 3, 64, 127]
        want = ob.recognise_pinned(self.w.ora, np.ascontiguousarray(self.pcm(v)[rows]), 2400, None, 0, 4096)
        slots = sr_b200.make_bank(want["ftr"])
        slots[want["status"] != 0] = 0xFF
        bad = oracle_diff({"slots": out["bank"][rows], "status": out["status"][rows]}, {"slots": slots, "status": want["status"]})
        al = ox.align()
        avg, score, anchor = al.average_bank(out["bank"], 4096, self.K, 118, 2)
        bad += oracle_diff({k: out[k] for k in ("avg", "score", "anchor")}, {"avg": avg, "score": score, "anchor": anchor})
        sel = [0, 5, 66, 127]
        a = np.ascontiguousarray(out["bank"][sel, :sr_b200.FTR_BYTES]).view(sr_b200.FTR_DTYPE).reshape(-1)
        b = np.ascontiguousarray(out["avg"][[(s // self.K) * self.K for s in sel], :sr_b200.FTR_BYTES]).view(sr_b200.FTR_DTYPE).reshape(-1)
        dis, path, plen = al.dtw_path(a, b, 118)
        bad += oracle_diff({k: out[k][sel] for k in ("dis", "path", "path_len")}, {"dis": dis, "path": path, "path_len": plen})
        return bad


class LongConnected(Job):
    """sr_mfcc_long_batch at U = 65 535 (up to 818 frames), then sr_connected_batch against a 128-slot bank (16-CTA
    clusters)"""
    name = "mfcc_long_connected"
    calls = ("sr_mfcc_long_batch", "sr_connected_batch")
    B, U, P, MW = 64, 65535, 4000, 24
    rows = (0, 9)

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank128, 128, 4096)
        self.inputs = []
        for v in range(2):
            pcm = self.w.pcm(self.B, self.U, 0xC6000000 + v, 3)
            rng = np.random.default_rng(0xC6 + v)
            seg = np.zeros((self.B, 2), np.uint32)
            for b in range(self.B):
                st = 0 if b % 4 == 0 else int(rng.integers(1, 20000))
                en = self.U if b % 2 == 0 else int(rng.integers(st + 200, self.U + 1))
                seg[b] = st, en
            atap = np.concatenate([self.w.po.noise_atap(pcm[b], 2400) for b in range(self.B)])
            self.inputs.append((pcm, seg, atap))

    def run(self, v):
        pcm, seg, atap = self.inputs[v]
        feat, frm = self.h.mfcc_long(pcm, seg, atap)
        words, n_words, total = self.h.connected(feat, frm, self.P, self.MW)
        return {"feat": feat, "frm_num": frm, "words": words, "n_words": n_words, "total": total}

    def oracle(self, v, out):
        pcm, seg, atap = self.inputs[v]
        rows = list(self.rows)
        feat, frm = ox.mfcc_long(self.w.ora, np.ascontiguousarray(pcm[rows]), seg[rows], atap[rows], ox.CONN_FRM_MAX)
        words, nw, total = ox.connected().connected(feat, frm, self.w.bank128, 128, 4096, self.P, self.MW)
        return oracle_diff({k: out[k][rows] for k in ("feat", "frm_num", "words", "n_words", "total")},
                            {"feat": feat, "frm_num": frm, "words": words, "n_words": nw, "total": total})


class Grammar(Job):
    """sr_recognise_connected_grammar_batch under a 4-digit PIN chain grammar, then sr_recognise_connected_batch (the
    loop grammar), on 3-word captures"""
    name = "connected_grammar"
    calls = ("sr_recognise_connected_grammar_batch", "sr_recognise_connected_batch")
    B, U, MW = 96, 16000, 8
    rows = (0, 17)
    PIN = sr_b200.chain_grammar(4, 0x3FF)

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank40, 40, 4096)

    def pcm(self, v):
        return self.w.pcm(self.B, self.U, 0xC7000000 + v, 3)

    def run(self, v):
        g = self.h.recognise_connected_grammar(self.pcm(v), self.PIN, 0, self.MW)
        c = self.h.recognise_connected(self.pcm(v), 3000, self.MW)
        return dict([("pin_" + k, a) for k, a in g.items()] + [("loop_" + k, a) for k, a in c.items()])

    def oracle(self, v, out):
        rows = list(self.rows)
        pcm = np.ascontiguousarray(self.pcm(v)[rows])
        g = ox.recognise_connected_grammar(self.w.ora, ox.grammar(), pcm, 2400, self.w.bank40, 40, 4096, self.PIN, 0, self.MW)
        c = ox.recognise_connected(self.w.ora, ox.connected(), pcm, 2400, self.w.bank40, 40, 4096, 3000, self.MW)
        want = dict([("pin_" + k, a) for k, a in g.items()] + [("loop_" + k, a) for k, a in c.items()])
        return oracle_diff({k: out[k][rows] for k in want}, want)


def _event_oracle(w, pcm, bank, T, out, streams):
    """segments, atap and the events of `streams` against the oracle, stage by stage"""
    bad = []
    ev = out["events"]
    for s in streams:
        atap = w.ora.noise_atap(pcm[s], 2400)
        seg = w.ora.vad(pcm[s], pcm.shape[1], atap).reshape(3, 2)
        bad += [("atap %d" % s, d) for d in [first_diff(out["atap"][s:s + 1].view(np.uint8), atap.view(np.uint8))] if d]
        bad += [("seg %d" % s, d) for d in [first_diff(out["seg"][s], seg)] if d]
        for e in ev[ev["stream"] == s]:
            k = int(e["segment"])
            f = w.ora.mfcc_batch(pcm[s:s + 1], seg[k].reshape(1, 2), atap)
            sc, _ = w.ora.dtw_batch(f, bank, T, 4096, check_sign=1)
            bi, bd = _argmin_rows(sc)
            got = tuple(int(e[q]) for q in ("start", "end", "frm_num", "best_idx", "best_dis", "cmd"))
            want = (int(seg[k, 0]), int(seg[k, 1]), int(f["frm_num"][0]), int(bi[0]), int(bd[0]), int(bi[0]) // 4)
            if got != want:
                bad.append(("event %d/%d" % (s, k), "%s != %s" % (got, want)))
    return bad


class StreamRagged(Job):
    """sr_streams_push_ragged: 40 streams fed ragged chunks (0 to 4 000 samples, one stream starting late); events sorted
    by (stream, segment), final segments and atap"""
    name = "stream_pool"
    calls = ("sr_streams_create", "sr_streams_destroy", "sr_streams_reset", "sr_streams_push_ragged", "sr_streams_segments",
             "sr_streams_pending")
    S, L = 40, 24000

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank8, 8, 4096)
        self.pool = sr_b200.StreamPool(self.h, self.S, self.L, 2400)
        self.pushes = []
        for v in range(2):
            pcm = self.w.pcm(self.S, self.L, 0xC8000000 + v, 3)
            rng = np.random.default_rng(0xC8 + v)
            pos, pushes = np.zeros(self.S, np.int64), []
            while (pos < self.L).any():
                lens = rng.choice([0, 1, 79, 80, 81, 160, 333, 800, 1601, 4000], self.S).astype(np.int64)
                lens[5] = 0 if len(pushes) < 10 else lens[5]
                lens = np.minimum(lens, self.L - pos)
                w = int(lens.max())
                if w == 0:
                    continue
                chunk = np.zeros((self.S, w), np.uint16)
                for s in range(self.S):
                    chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
                pushes.append((chunk, lens.astype(np.uint32)))
                pos += lens
            self.pushes.append(pushes)

    def close(self):
        self.pool.close()
        super().close()

    def run(self, v):
        self.pool.reset()
        events = []
        for chunk, lens in self.pushes[v]:
            events += self.pool.push_ragged(chunk, lens)
        assert self.pool.pending() == 0
        seg, atap = self.pool.segments()
        return {"events": events_array(events), "seg": seg, "atap": atap}

    def oracle(self, v, out):
        return _event_oracle(self.w, self.w.pcm(self.S, self.L, 0xC8000000 + v, 3), self.w.bank8, 8, out, (0, 5, 39))


class StreamGroup(Job):
    """sr_stream_group of two handles on device 0: 37 streams, lock-step pushes of 800 samples"""
    name = "stream_group"
    calls = ("sr_stream_group_create", "sr_stream_group_destroy", "sr_stream_group_reset", "sr_stream_group_push",
             "sr_stream_group_segments")
    S, L = 37, 24000

    def open(self):
        hs = [self.handle(), self.handle()]
        for h in hs:
            h.set_bank(self.w.bank8, 8, 4096)
        self.pool = sr_b200.StreamPool(hs, self.S, self.L, 2400)

    def close(self):
        self.pool.close()
        super().close()

    def run(self, v):
        self.pool.reset()
        pcm = self.w.pcm(self.S, self.L, 0xC9000000 + v, 3)
        events = []
        for n0 in range(0, self.L, 800):
            events += self.pool.push(np.ascontiguousarray(pcm[:, n0:n0 + 800]))
        seg, atap = self.pool.segments()
        return {"events": events_array(events), "seg": seg, "atap": atap}

    def oracle(self, v, out):
        return _event_oracle(self.w, self.w.pcm(self.S, self.L, 0xC9000000 + v, 3), self.w.bank8, 8, out, (0, 18, 19, 36))


class LongForm(Job):
    """sr_vad_long_batch and sr_recognise_long_batch on host PCM with ragged lens (poison past them), then
    sr_recognise_long_batch_dev on the same recordings on a torch stream of the job's own; device outputs prefilled"""
    name = "long_form"
    calls = ("sr_vad_long_batch", "sr_recognise_long_batch", "sr_recognise_long_batch_dev")
    B, U, MS = 6, 150001, 16

    def open(self):
        import torch
        self.torch = torch
        self.h = self.handle()
        self.h.set_bank(self.w.bank40, 40, 4096)
        self.st = torch.cuda.Stream(torch.device("cuda:0"))
        self.h.set_stream(self.st.cuda_stream)
        self.inputs = []
        for v in range(2):
            pcm = ox.synth_long(self.B, self.U, 0xCC000000 + v)
            lens = np.array([self.U, 161, 90000 + v, 2399, 120001, self.U - 80 * v], np.uint32)
            for b, n in enumerate(lens):
                pcm[b, n:] = np.where(np.arange(self.U - n) % 2, 4095, 0)
            self.inputs.append((pcm, lens))
        with torch.cuda.stream(self.st):
            self.dev = [(torch.from_numpy(p.view(np.int16)).to("cuda:0"), torch.from_numpy(n.view(np.int32)).to("cuda:0"))
                        for p, n in self.inputs]
            self.out = {k: torch.empty(self.B * n, dtype=torch.uint8, device="cuda:0")
                        for k, n in (("atap", 12), ("n_segs", 4), ("segs", 28 * self.MS))}
        self.st.synchronize()

    def run(self, v):
        pcm, lens = self.inputs[v]
        vad = self.h.vad_long_batch(pcm, self.MS, 2400, lens)
        rec = self.h.recognise_long_batch(pcm, self.MS, 2400, lens)
        d_pcm, d_lens = self.dev[v]
        with self.torch.cuda.stream(self.st):
            for k, t in self.out.items():
                t.fill_(0 if k == "atap" else 0x5A)             # atap is in / out: rows noise_atap skips keep zeros
            self.h.recognise_long_batch_dev(d_pcm.data_ptr(), self.U, self.B, d_lens.data_ptr(), 2400, self.MS,
                                            *(self.out[k].data_ptr() for k in ("atap", "n_segs", "segs")))
            self.h.sync()
            o = {k: t.cpu().numpy() for k, t in self.out.items()}
        return {"vad_atap": vad["atap"], "vad_n_segs": vad["n_segs"], "seg_off": vad["seg_off"], "atap": rec["atap"],
                "n_segs": rec["n_segs"], "segs": rec["segs"], "dev_atap": o["atap"].view(sr_b200.ATAP_DTYPE),
                "dev_n_segs": o["n_segs"].view(np.uint32), "dev_segs": o["segs"].view(ox.LONG_SEG_DTYPE).reshape(self.B, self.MS)}

    def oracle(self, v, out):
        pcm, lens = self.inputs[v]
        want = ox.recognise_long(ox.long_oracle(), self.w.po, pcm, 2400, self.w.bank40, 40, 4096, self.MS, lens)
        k = np.arange(self.MS)[None, :] < np.minimum(want["n_segs"], self.MS)[:, None]
        got = {"vad_atap": out["vad_atap"], "vad_n_segs": out["vad_n_segs"], "seg_off": out["seg_off"][k],
               "atap": out["atap"], "n_segs": out["n_segs"], "segs": out["segs"][k], "dev_atap": out["dev_atap"],
               "dev_n_segs": out["dev_n_segs"], "dev_segs": out["dev_segs"][k]}
        seg_off = np.stack([want["segs"]["start"], want["segs"]["end"]], -1)[k]
        return diff_outputs(got, {"vad_atap": want["atap"], "vad_n_segs": want["n_segs"], "seg_off": seg_off, "atap": want["atap"],
                                  "n_segs": want["n_segs"], "segs": want["segs"][k], "dev_atap": want["atap"],
                                  "dev_n_segs": want["n_segs"], "dev_segs": want["segs"][k]})


class _SharedBank:
    """one read-only device copy of the 200-slot bank that both bank_dev jobs borrow"""
    t = None

    @classmethod
    def ptr(cls, w):
        if cls.t is None:
            import torch
            cls.t = torch.from_numpy(w.bank200.reshape(-1).copy()).to("cuda:0")
            torch.cuda.synchronize()
        return cls.t.data_ptr()


class BankDevRecognise(Job):
    """sr_recognise_batch against the shared device bank (sr_set_bank_dev)"""
    name = "bank_dev_recognise"
    calls = ("sr_set_bank_dev", "sr_recognise_batch")
    B, U = 1024, 8000
    rows = (0, 511, 1023)

    def open(self):
        self.h = self.handle()
        self.h.set_transport(0)
        self.h.set_bank_dev(_SharedBank.ptr(self.w), 200, 4096)

    def run(self, v):
        return self.h.recognise(self.w.pcm(self.B, self.U, 0xCA000000 + v))

    def oracle(self, v, out):
        rows = list(self.rows)
        pcm = np.ascontiguousarray(self.w.pcm(self.B, self.U, 0xCA000000 + v)[rows])
        want = ob.recognise_pinned(self.w.ora, pcm, 2400, self.w.bank200, 200, 4096)
        return oracle_diff({k: out[k][rows] for k in want}, want)


class BankDevDtw(Job):
    """sr_dtw_batch (static greedy kernel) against the same shared device bank"""
    name = "bank_dev_dtw"
    calls = ("sr_set_bank_dev", "sr_dtw_batch")
    B = 2000
    rows = (0, 1999)

    def open(self):
        self.h = self.handle()
        self.h.set_dtw_variant(0)
        self.h.set_bank_dev(_SharedBank.ptr(self.w), 200, 4096)

    def fin(self, v):
        return sr_b200.synth_ftr_host(self.B, 0xCB000000 + v, 20, 119).view(sr_b200.FTR_DTYPE).reshape(-1)

    def run(self, v):
        score, bi, bd = self.h.dtw(self.fin(v), flags=sr_b200.DTW_CHECK_SIGN)
        return {"score": score, "best_idx": bi, "best_dis": bd}

    def oracle(self, v, out):
        rows = list(self.rows)
        sc, _ = self.w.ora.dtw_batch(np.ascontiguousarray(self.fin(v)[rows]), self.w.bank200, 200, 4096, check_sign=1)
        bi, bd = _argmin_rows(sc)
        return oracle_diff({k: out[k][rows] for k in ("score", "best_idx", "best_dis")},
                            {"score": sc, "best_idx": bi, "best_dis": bd})


class LongGrammar(Job):
    """sr_recognise_long_grammar_batch on ragged lens (one past 65 535 samples) under a 5-state PIN chain and then a
    2-state alternation, so the record workspace changes size between inputs; max_segs below n_segs, atap NULL on input
    1; then sr_connected_grammar_segs_batch on a small flat segment table"""
    name = "long_grammar"
    calls = ("sr_recognise_long_grammar_batch", "sr_connected_grammar_segs_batch")
    B, U, P, MS, MW = 5, 120000, 1000, 4, 48
    GRAMS = (sr_b200.chain_grammar(4, 0x3FF), (2, 3, [(0, 1, 0x55), (1, 0, 0x2AA), (1, 1, 0x1)]))

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank40, 40, 4096)
        self.inputs = []
        for v in range(2):
            pcm = ox.synth_long(self.B, self.U, 0xCD000000 + v)
            lens = np.array([self.U, 70001 + v, 2399, 40000, self.U - 160 * v], np.uint32)
            rng = np.random.default_rng(0xCD + v)
            seg_frm = np.array([30, 0, 119, 5, 64 + v, 818], np.uint32)
            feat = rng.integers(-3000, 3001, (int(seg_frm.sum()), 12)).astype(np.int16)
            self.inputs.append((pcm, lens, feat, np.array([0, 2, 3, 6], np.uint32), seg_frm))

    def run(self, v):
        pcm, lens, feat, seq_seg, seg_frm = self.inputs[v]
        g = self.GRAMS[v]
        want = sr_b200.LONG_GRAM_FIELDS if v == 0 else tuple(k for k in sr_b200.LONG_GRAM_FIELDS if k != "atap")
        out = self.h.recognise_long_grammar(pcm, g, self.P, self.MS, self.MW, 2400, lens, want=want)
        w, nw, tot = self.h.connected_grammar_segs(feat, seq_seg, seg_frm, g, self.P, self.MW)
        out.update({"segs_words": w, "segs_n_words": nw, "segs_total": tot})
        return out

    def oracle(self, v, out):
        pcm, lens, feat, seq_seg, seg_frm = self.inputs[v]
        g, lg = self.GRAMS[v], ox.long_grammar()
        want = ox.recognise_long_grammar(ox.long_oracle(), self.w.po, lg, pcm, 2400, self.w.bank40, 40, 4096, g, self.P,
                                         self.MS, self.MW, lens)
        if v == 1:
            del want["atap"]
        assert (want["n_segs"] > self.MS).any() and (want["n_words"] > 0).any()
        w, nw, tot = lg.decode_segs(feat, seq_seg, seg_frm, self.w.bank40, 40, 4096, g, self.P, self.MW)
        want.update({"segs_words": w, "segs_n_words": nw, "segs_total": tot})
        return diff_outputs(out, want)


class LongStream(Job):
    """sr_long_streams_*: a pool of 24 streams made and destroyed in every repetition, ragged pushes of 0-1 600 samples
    (every third with a caller buffer of 2 events, so events queue) and a lock-step push, pending / fetch, a subset
    reset with the queue drained, then more pushes; events sorted by (stream, segment), state(), max_events, ring_len"""
    name = "long_stream"
    calls = ("sr_long_streams_create", "sr_long_streams_destroy", "sr_long_streams_reset", "sr_long_streams_push",
             "sr_long_streams_push_ragged", "sr_long_streams_fetch", "sr_long_streams_pending",
             "sr_long_streams_max_events", "sr_long_streams_ring_len", "sr_long_streams_state")
    S, L, MC = 24, 36000, 1600
    RESET = np.arange(24) % 5 == 1                    # the streams restarted halfway

    def open(self):
        self.h = self.handle()
        self.h.set_bank(self.w.bank8, 8, 4096)
        self.inputs = []
        for v in range(2):
            pcm = ox.synth_long(self.S, self.L, 0xCE000000 + v)
            rng = np.random.default_rng(0xCE + v)
            pos, pushes = np.zeros(self.S, np.int64), []
            while (pos < self.L).any():
                lens = rng.choice([0, 1, 79, 80, 81, 333, 800, self.MC], self.S).astype(np.int64)
                lens = np.minimum(lens, self.L - pos)
                if len(pushes) % 7 == 3:
                    lens[:] = min(640, int((self.L - pos).min()))              # a lock-step push
                chunk = np.zeros((self.S, max(1, int(lens.max()))), np.uint16)
                for s in range(self.S):
                    chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
                pushes.append((chunk, lens.astype(np.uint32), pos.copy()))
                pos += lens
            self.inputs.append((pcm, pushes))

    def run(self, v):
        pcm, pushes = self.inputs[v]
        pool = sr_b200.LongStreamPool(self.h, self.S, self.MC, 2400)
        try:
            before, after, queued, half = [], [], [], len(pushes) // 2
            for i, (chunk, lens, _) in enumerate(pushes):
                evs = before if i < half else after
                m = 2 if i % 3 == 2 else None
                if (lens == lens[0]).all() and lens[0]:
                    evs += pool.push(np.ascontiguousarray(chunk[:, :lens[0]]), max_events=m)
                else:
                    evs += pool.push_ragged(chunk, lens, max_events=m)
                queued.append(pool.pending())
                if i == half - 1:
                    evs += pool.fetch(max_events=pool.pending())    # all of it: the reset must find the queue empty
                    assert pool.pending() == 0
                    pool.reset(self.RESET.astype(np.uint8))
            after += pool.fetch(max_events=pool.pending())
            st = pool.state()
            return {"before": events_array(before), "after": events_array(after), "n_recv": st["n_recv"],
                    "n_closed": st["n_closed"], "open_start": st["open_start"], "atap": st["atap"],
                    "queued": np.array(queued, np.uint32),
                    "sizes": np.array([pool.max_events, pool.ring_len, pool.pending()], np.uint32)}
        finally:
            pool.close()

    def _closed(self, x):
        """sr_recognise_long_batch of one stream's samples from the oracles: (closed records, open start, atap)"""
        r = ox.recognise_long(ox.long_oracle(), self.w.po, np.ascontiguousarray(x[None, :]), 2400, self.w.bank8, 8, 4096,
                              len(x) // 1520 + 4)
        recs = [tuple(int(q) for q in rec) for rec in r["segs"][0, :int(r["n_segs"][0])].tolist()]
        op = recs[-1][0] if recs and recs[-1][2] == 1 else 0xFFFFFFFF
        return [t for t in recs if t[2] != 1], op, r["atap"][0].tobytes()

    def oracle(self, v, out):
        pcm, pushes = self.inputs[v]
        cut = pushes[len(pushes) // 2][2]                 # each stream's sample count at the reset
        E = -(-(-(-(self.MC + 2400) // 80)) // 19)        # the header's bound, c = n_len
        bad = diff_outputs({"sizes": out["sizes"]},
                           {"sizes": np.array([self.S * E, -(-(10561 + self.MC) // 80) * 80, 0], np.uint32)})
        if out["queued"].max() == 0:
            bad.append(("queued", "no push left events queued"))
        fields = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")
        for s in (0, 1, 6, self.S - 1):
            pre = self._closed(pcm[s, :int(cut[s])])[0]
            x = pcm[s, int(cut[s]):] if self.RESET[s] else pcm[s]
            closed, op, atap = self._closed(x)
            for part, want in (("before", pre), ("after", closed if self.RESET[s] else closed[len(pre):])):
                ev = out[part][out[part]["stream"] == s]
                got = [tuple(int(e[k]) for k in fields) for e in ev]
                first = 0 if part == "before" or self.RESET[s] else len(pre)
                if got != want or ev["segment"].tolist() != list(range(first, first + len(ev))):
                    bad.append(("%s events of stream %d" % (part, s), "%d events, %d closed records" % (len(got), len(want))))
            st = (int(out["n_recv"][s]), int(out["n_closed"][s]), int(out["open_start"][s]), out["atap"][s].tobytes())
            if st != (len(x), len(closed), op, atap):
                bad.append(("state of stream %d" % s, "%s" % (st[:3],)))
        return bad


JOBS = (RecognisePacked, RecogniseDevBand, DtwDynamic, GeomB, EnrolAverageAlign, LongConnected, Grammar, StreamRagged,
        StreamGroup, BankDevRecognise, BankDevDtw, LongForm, LongGrammar, LongStream)
RECREATED = "dtw_dynamic"                # the job whose thread destroys its handle and makes a new one halfway through

# sr_* entry points of the headers that no job runs, each with the reason
EXCLUDED = {
    "sr_comm_unique_id": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_create": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_destroy": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_rank": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_world": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_nccl_version": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_comm_wait": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_allgather_dev": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_recognise_batch_dev_allgather": "NCCL: a communicator of its own; test_decision_paths.py runs it on one rank",
    "sr_recognise_batch_multi": "requires handles on different devices",
    "sr_stream_group_push_ragged": "the group's ragged push is the pool's ragged push per shard; the stream_pool job runs it",
    "sr_streams_push": "the lock-step push is a ragged push with equal lengths; stream_pool and stream_group run both forms",
    "sr_streams_fetch": "only hands out queued events; no queue forms with events buffers of 3 * n_streams",
    "sr_noise_atap_batch": "its kernel is the recognise path's first launch (tag 0), run by every recognise job",
    "sr_vad_batch": "its kernel is the recognise path's first launch (tag 0), run by every recognise job",
    "sr_mfcc_batch": "its kernel runs in every recognise job; the subprocess start-up test calls it from 8 threads",
    "sr_noise_atap_batch_dev": "device-pointer form of the recognise front end; recognise_dev_band runs the same kernel",
    "sr_vad_batch_dev": "device-pointer form of the recognise front end; recognise_dev_band runs the same kernel",
    "sr_mfcc_batch_dev": "device-pointer form of the recognise front end; recognise_dev_band runs the same kernel",
    "sr_dtw_batch_dev": "device-pointer form of sr_dtw_batch, which dtw_dynamic and bank_dev_dtw run",
    "sr_vad_long_batch_dev": "its three launches are the first of sr_recognise_long_batch_dev, which long_form runs",
    "sr_get_mdl_batch": "test-hook kernel of the unused get_mdl; stateless, no workspace of its own",
    "sr_connected_grammar_batch": "kernel-level form of sr_recognise_connected_grammar_batch, which connected_grammar runs",
    "sr_fft_mag_batch": "stateless test-hook kernel; the drop-in fft() runs it from 8 threads",
    "sr_get_dis_batch": "stateless test-hook kernel of get_dis",
    "sr_dtw_limit_batch": "stateless; the drop-in dtw_limit() runs it from 8 threads",
    "sr_fft_raw_batch": "stateless test-hook kernel",
    "sr_debug_fft_raw_n": "stateless test-hook kernel",
    "sr_debug_sqrt_mismatches": "stateless test-hook kernel",
    "sr_debug_log100_mismatches": "stateless test-hook kernel",
    "sr_debug_mag10_mismatches": "stateless test-hook kernel",
    "sr_debug_pack12_host": "host only, no handle",
    "sr_debug_unpack12": "stateless test-hook kernel; recognise_packed runs the expander",
    "sr_set_labels": "host-side table of the handle; no device state",
    "sr_label": "host-side table of the handle; no device state",
    "sr_labels_batch": "host-side table of the handle; no device state",
    "sr_bind_thread_to_device": "changes the calling thread's CPU affinity, which would leak into the test process",
    "sr_device_numa_node": "reads the topology only",
    "sr_host_numa_node": "reads the topology only",
    "sr_device_count": "reads the device count only",
    "sr_abi_version": "a constant",
    "sr_last_error": "checked per thread by test_dropins_keep_per_thread_state",
    "sr_host_alloc": "sr_host_alloc_dev falls back to it on single-node hosts; allocated and freed in a loop during the run",
}
# entry points the tests of this file call besides the job table
OTHER_CALLS = ("sr_create", "sr_destroy", "sr_use_own_stream", "sr_host_alloc_dev", "sr_host_free", "sr_timing_enable",
               "sr_timing_collect", "sr_launch_count")


def header_entry_points():
    names = set()
    for hdr in HEADERS:
        src = re.sub(r"/\*.*?\*/", " ", open(hdr).read(), flags=re.S)
        names |= set(re.findall(r"\b(sr_\w+)\s*\(", src))
    return sorted(names)


def test_every_entry_point_is_in_the_job_table_or_excluded():
    """a new sr_* entry point of the headers cannot skip the concurrency check without an entry here"""
    names = header_entry_points()
    assert len(names) > 60 and "sr_recognise_batch" in names and "sr_connected_grammar_batch" in names, names
    assert "sr_vad_long_batch_dev" in names, names
    newer = {"sr_connected_grammar_segs_batch", "sr_recognise_long_grammar_batch"} | {
        "sr_long_streams_" + n for n in ("create", "destroy", "reset", "push", "push_ragged", "fetch", "pending", "max_events",
                                         "ring_len", "state")}
    assert newer <= set(names), newer - set(names)
    assert {os.path.basename(h) for h in HEADERS} >= {"speech_recog.h", "sr_long.h", "sr_long_grammar.h", "sr_long_stream.h"}
    covered = {c for j in JOBS for c in j.calls} | set(OTHER_CALLS)
    assert not (covered & set(EXCLUDED)), covered & set(EXCLUDED)
    missing = [n for n in names if n not in covered and n not in EXCLUDED]
    assert not missing, "entry points neither in the job table nor excluded: %s" % missing
    lib_syms = set(re.findall(r"\b(sr_\w+)\b", open(SYNTH_HEADER).read()))
    stale = [n for n in (covered | set(EXCLUDED)) if n not in names and n not in lib_syms]
    assert not stale, "listed but not declared: %s" % stale
    assert len({j.name for j in JOBS}) == len(JOBS) and RECREATED in {j.name for j in JOBS}
    assert all(j.calls and j.__doc__ for j in JOBS)


# ---- the GPU tests -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def world():
    return World()


def _rep(job, v):
    """one repetition of input variant v: (outputs, launches, timing tags per handle, (t0, t1))"""
    for h in job.hs:
        h.timing_collect()
    l0 = [h.launch_count() for h in job.hs]
    t0 = time.perf_counter()
    out = job.run(v)
    t1 = time.perf_counter()
    n = sum(h.launch_count() - a for h, a in zip(job.hs, l0)) - job.varying_launches()
    tags = [[t for t, _ in h.timing_collect()] for h in job.hs]
    return out, n, tags, (t0, t1)


@pytest.fixture(scope="module")
def baseline(world):
    """every job alone on fresh handles, both input variants: {name: [(outputs, launches, tags, oracle mismatches,
    seconds)] per variant}"""
    base = {}
    for J in JOBS:
        job = J(world)
        try:
            base[J.name] = []
            for v in range(2):
                out, n, tags, (t0, t1) = _rep(job, v)
                base[J.name].append((out, n, tags, job.oracle(v, out), t1 - t0))
        finally:
            job.close()
    return base


@pytest.mark.gpu
def test_serial_baseline_matches_the_oracles(baseline):
    """each job run alone agrees with its oracle on a sample of every output, for both input variants, so the
    concurrent run is compared with results that are right, not only with the GPU agreeing with itself"""
    print("serial repetition ms: " + ", ".join("%s %.1f/%.1f" % (n, 1e3 * r[0][4], 1e3 * r[1][4]) for n, r in baseline.items()))
    bad = [(name, v, k, d) for name, runs in baseline.items() for v, r in enumerate(runs) for k, d in r[3]]
    assert not bad, bad
    for name, runs in baseline.items():
        assert runs[0][1] > 0, name
    st = baseline["stream_pool"][0][0]["events"]
    assert len(set(st["stream"].tolist())) == StreamRagged.S and (st["status"] == 0).mean() > 0.5
    assert (baseline["recognise_packed"][0][0]["status"] == 0).mean() > 0.95
    pin = baseline["connected_grammar"][0][0]
    assert (pin["pin_n_words"][pin["pin_status"] == 0] == 4).all() and (pin["pin_status"] == 0).sum() > 16
    lc = baseline["mfcc_long_connected"][0][0]
    assert (lc["frm_num"] == ox.CONN_FRM_MAX).sum() == LongConnected.B // 4 and (lc["n_words"][lc["frm_num"] > 0] >= 1).all()
    tags = baseline["enrol_average_path"][0][2][0]
    assert {ALIGN, AVG_UPDATE} <= set(tags) and GRAM in baseline["connected_grammar"][0][2][0]
    assert CONN in baseline["mfcc_long_connected"][0][2][0] and DTW_BAND in baseline["recognise_dev_band"][0][2][0]


def _compare(name, rep, v, got, base, n, tags):
    want, n0, tags0 = base[v][:3]
    msgs = ["%s rep %d (input %d): field %s: %s" % (name, rep, v, k, d) for k, d in diff_outputs(got, want)]
    if n != n0:
        msgs.append("%s rep %d: %d launches, %d alone" % (name, rep, n, n0))
    if tags != tags0:
        msgs.append("%s rep %d: timing tags %s, alone %s" % (name, rep, tags, tags0))
    return msgs


def _run_threads(targets, timeout):
    """run each (name, callable) on a thread of its own and join every one; [(name, traceback)] of those that raised"""
    errors = []

    def wrap(name, f):
        def body():
            try:
                f()
            except BaseException:
                errors.append((name, traceback.format_exc()))
        return body
    ts = [threading.Thread(target=wrap(n, f), name=n) for n, f in targets]
    for t in ts:
        t.start()
    deadline = time.time() + timeout
    for t in ts:
        t.join(max(1.0, deadline - time.time()))
    alive = [t.name for t in ts if t.is_alive()]
    assert not alive, "threads still running after %d s: %s" % (timeout, alive)
    return errors


def _max_overlap(intervals):
    """the largest number of different jobs inside a repetition at the same moment"""
    pts = sorted([(t0, 1, j) for j, t0, t1 in intervals] + [(t1, -1, j) for j, t0, t1 in intervals], key=lambda p: (p[0], p[1]))
    inside, best = {}, 0
    for _, d, j in pts:
        inside[j] = inside.get(j, 0) + d
        best = max(best, sum(1 for c in inside.values() if c > 0))
    return best


@pytest.mark.gpu
def test_concurrent_handles_equal_the_serial_baseline(world, baseline):
    """every job on its own handle and thread, started together behind a barrier, R repetitions each, alternating
    between the two inputs; meanwhile two threads allocate and free pinned host memory, and one job destroys its handle
    and makes a new one halfway through. Every repetition equals the serial baseline bit for bit, with the same launches
    and timing tags per handle"""
    jobs = [J(world) for J in JOBS]
    n_alloc = 2
    bar = threading.Barrier(len(jobs) + n_alloc, timeout=300)
    jobs_done = threading.Event()
    reports, intervals, allocs = {}, [], [0] * n_alloc
    lock = threading.Lock()

    def run_job(job):
        def body():
            msgs = []
            bar.wait()
            for rep in range(R):
                if job.name == RECREATED and rep == R // 2:
                    job.close()                                   # the others are mid-call: the per-device tables stay
                    job.open()
                out, n, tags, (t0, t1) = _rep(job, rep % 2)
                msgs += _compare(job.name, rep, rep % 2, out, baseline[job.name], n, tags)
                with lock:
                    intervals.append((job.name, t0, t1))
            reports[job.name] = msgs
        return body

    def alloc_loop(k):
        def body():
            L = sr_b200.lib()
            rng = np.random.default_rng(k)
            bar.wait()
            while not jobs_done.is_set():
                nb = int(rng.integers(1, 64)) << 16
                p = L.sr_host_alloc_dev(0, nb)
                assert p, "sr_host_alloc_dev(0, %d) returned NULL" % nb
                a = np.frombuffer((C.c_uint8 * nb).from_address(p), np.uint8)
                a[::4096] = k + 1
                ok = bool((a[::4096] == k + 1).all())
                del a
                L.sr_host_free(C.c_void_p(p))
                assert ok
                allocs[k] += 1
        return body

    def all_jobs():
        try:
            errs = _run_threads([(j.name, run_job(j)) for j in jobs], timeout=900)
            assert not errs, "\n".join("%s:\n%s" % e for e in errs)
        finally:
            jobs_done.set()

    try:
        errs = _run_threads([("jobs", all_jobs)] + [("alloc%d" % k, alloc_loop(k)) for k in range(n_alloc)], timeout=960)
    finally:
        jobs_done.set()
        for j in jobs:
            j.close()
    assert not errs, "\n".join("%s:\n%s" % e for e in errs)
    msgs = [m for j in jobs for m in reports.get(j.name, ["%s: no report" % j.name])]
    assert not msgs, "\n".join(msgs[:40])
    assert min(allocs) > 0, allocs
    stats = jobs[0].stats
    assert jobs[0].name == "recognise_packed" and len(stats) == R and all(p + q == 4 for p, q, _ in stats), stats
    if _cpus() >= 8:                                      # with fewer CPUs the library creates no packer pool
        assert all(p >= 1 for p, _, _ in stats), stats
    overlap = _max_overlap(intervals)
    print("jobs inside a repetition at once: at most %d of %d" % (overlap, len(jobs)))
    assert overlap >= 3, "at most %d jobs ran at the same moment: nothing ran concurrently (%s)" % (overlap, intervals)


@pytest.mark.gpu
def test_one_handle_across_caller_streams(world):
    """the same sr_recognise_batch_dev on one handle five times: on torch stream S1; after sr_sync on S2; on its own
    stream (sr_use_own_stream); on the legacy default stream (sr_set_stream(NULL)); on S1 again while another handle's
    job runs. All five equal, outputs prefilled before each call"""
    import torch
    job = RecogniseDevBand(world)
    other = DtwDynamic(world)
    h = job.h
    s1, s2 = torch.cuda.Stream(torch.device("cuda:0")), torch.cuda.Stream(torch.device("cuda:0"))
    torch.cuda.synchronize()

    def once(v=0):
        for t in job.out.values():
            t.fill_(0x5A)
        torch.cuda.synchronize()
        h.recognise_dev(job.pcm[v].data_ptr(), job.U, job.B, 2400, **{k: t.data_ptr() for k, t in job.out.items()})
        h.sync()
        return job._host()

    try:
        h.set_match(sr_b200.DTW_BAND, 10)
        res = []
        h.set_stream(s1.cuda_stream)
        res.append(("S1", once()))
        h.sync()
        h.set_stream(s2.cuda_stream)
        res.append(("S2", once()))
        h.use_own_stream()
        res.append(("own stream", once()))
        h.set_stream(None)
        res.append(("legacy default stream", once()))
        h.set_stream(s1.cuda_stream)
        got = {}

        def ours():
            time.sleep(0.005)
            got["x"] = once()
        errs = _run_threads([("other", lambda: [_rep(other, v % 2) for v in range(2)]), ("ours", ours)], timeout=300)
        assert not errs, errs
        res.append(("S1 beside another handle", got["x"]))
    finally:
        job.close()
        other.close()
    ref = res[0][1]
    assert (ref["status"] == 0).mean() > 0.9
    for what, out in res[1:]:
        assert not diff_outputs(out, ref), (what, diff_outputs(out, ref))


# the drop-ins: 8 threads at once, each with its own (I, M), frame and failure
N_DROPIN = 8
FAILS = (("sr_set_match", lambda L, h: L.sr_set_match(h, sr_b200.DTW_BAND, -1)),
         ("sr_set_geometry", lambda L, h: L.sr_set_geometry(h, 7)),
         ("sr_set_dtw_variant", lambda L, h: L.sr_set_dtw_variant(h, 5)),
         ("sr_set_transport", lambda L, h: L.sr_set_transport(h, 9)),
         ("sr_timing_collect", lambda L, h: L.sr_timing_collect(h, None, None, 0, None)),
         ("sr_create", lambda L, h: L.sr_create(9999, C.byref(C.c_void_p()))),
         ("sr_set_labels", lambda L, h: L.sr_set_labels(h, None, 3, 4)),
         ("sr_dtw_path_batch", lambda L, h: L.sr_dtw_path_batch(h, None, None, 0, -1, None, None, None)))


@pytest.mark.gpu
def test_dropins_keep_per_thread_state(world):
    """dtw_limit() reads the (I, M) of the calling thread's last dtw(), fft() returns a buffer of the calling thread, and
    sr_last_error(NULL) the calling thread's last failure -- while 7 other threads call the same functions"""
    L = sr_b200.lib()
    h0 = sr_b200.Handle(0)
    grid = np.array([(x, y) for x in range(0, 122) for y in range(0, 122)], np.uint16)
    xs, ys = np.ascontiguousarray(grid[:, 0]), np.ascontiguousarray(grid[:, 1])
    ctx = []
    for i in range(N_DROPIN):
        f = sr_b200.synth_ftr_host(2, 0xD0000 + i, 10, 119).view(sr_b200.FTR_DTYPE).reshape(-1).copy()
        f["frm_num"][0], f["frm_num"][1] = 12 + 13 * i, 119 - 9 * i            # (I, M) of this thread
        I, M = np.full(len(grid), f["frm_num"][0], np.uint16), np.full(len(grid), f["frm_num"][1], np.uint16)
        lim = np.zeros(len(grid), np.uint8)
        assert L.sr_dtw_limit_batch(h0._h, *[a.ctypes.data_as(C.c_void_p) for a in (xs, ys, I, M)], len(grid),
                                    lim.ctypes.data_as(C.c_void_p)) == 0
        d = L.dtw(f[0:1].ctypes.data_as(C.c_void_p), f[1:2].ctypes.data_as(C.c_void_p))
        frame = np.random.default_rng(i).integers(-2000, 2000, 160 + 100 * i).astype(np.int16)
        p = L.fft(frame.ctypes.data_as(C.c_void_p), len(frame))
        spec = np.ctypeslib.as_array(p, shape=(1024,)).copy()
        assert np.array_equal(spec[:512], world.ora.fft_mag(frame.reshape(1, -1))[0])
        ctx.append(dict(f=f, lim=lim, dtw=d, frame=frame, spec=spec))
    # each thread asks at lattice points where another thread's (I, M) gives a different answer
    for i, c in enumerate(ctx):
        c["pts"] = np.nonzero(np.any([c["lim"] != o["lim"] for o in ctx if o is not c], axis=0))[0]
        assert len(c["pts"]) >= 20, (i, len(c["pts"]))
    msgs0 = []
    for name, fail in FAILS:
        assert fail(L, h0._h) != 0, name
        msgs0.append(L.sr_last_error(None))
    assert len(set(msgs0)) == len(FAILS), msgs0
    h0.close()

    bar = threading.Barrier(N_DROPIN, timeout=120)
    ptrs, bad = [set() for _ in range(N_DROPIN)], []
    stop = [False]

    def body(i):
        def f():
            c = ctx[i]
            h = sr_b200.Handle(0)
            rng = np.random.default_rng(100 + i)
            a, b = c["f"][0:1].ctypes.data_as(C.c_void_p), c["f"][1:2].ctypes.data_as(C.c_void_p)
            fr = c["frame"].ctypes.data_as(C.c_void_p)
            try:
                # last error: the failures happen one thread after another, then every thread reads its own
                for rnd in range(3):
                    k = (i + rnd) % len(FAILS)
                    for turn in range(N_DROPIN):
                        bar.wait()
                        if turn == i:
                            FAILS[k][1](L, h._h)
                    bar.wait()
                    got = L.sr_last_error(None)
                    if got != msgs0[k]:
                        bad.append("thread %d round %d: sr_last_error(NULL) = %r, its own failure %r" % (i, rnd, got, msgs0[k]))
                    bar.wait()
                    if bad:
                        stop[0] = True
                    bar.wait()
                    if stop[0]:
                        return
                # then everything at once
                for it in range(40):
                    d = L.dtw(a, b)
                    if d != c["dtw"]:
                        bad.append("thread %d it %d: dtw = %d, alone %d" % (i, it, d, c["dtw"]))
                    for q in rng.choice(c["pts"], 6):
                        r = L.dtw_limit(int(grid[q, 0]), int(grid[q, 1]))
                        if r != c["lim"][q]:
                            bad.append("thread %d it %d: dtw_limit%s = %d, sr_dtw_limit_batch of its own (I, M) %d"
                                       % (i, it, tuple(grid[q]), r, c["lim"][q]))
                    p = L.fft(fr, len(c["frame"]))
                    ptrs[i].add(C.addressof(p.contents))
                    spec = np.ctypeslib.as_array(p, shape=(1024,)).copy()
                    if not np.array_equal(spec, c["spec"]):
                        bad.append("thread %d it %d: fft: %s" % (i, it, first_diff(spec, c["spec"])))
                    k = (i + it) % len(FAILS)
                    FAILS[k][1](L, h._h)
                    got = L.sr_last_error(None)
                    if got != msgs0[k]:
                        bad.append("thread %d it %d: sr_last_error(NULL) = %r, its own failure %r" % (i, it, got, msgs0[k]))
                bar.wait()                                        # every thread's fft buffer is alive until all have finished
            finally:
                h.close()
        return f

    errs = _run_threads([("dropin%d" % i, body(i)) for i in range(N_DROPIN)], timeout=600)
    assert not errs, "\n".join("%s:\n%s" % e for e in errs)
    assert not bad, "\n".join(bad[:20])
    assert all(len(p) == 1 for p in ptrs), "fft() returned several buffers to one thread: %s" % ptrs
    assert len(set.union(*ptrs)) == N_DROPIN, "fft() buffers shared between threads: %s" % ptrs


_STARTUP = r"""
import sys, threading
sys.path[:0] = [%r, %r]
import numpy as np
import oracle_bind as ob
import sr_b200
po = ob.port()
N, B, U = 8, 24, 8000
rng = np.random.default_rng(7)
case = []
for i in range(N):
    pcm = rng.integers(0, 4096, (B, U)).astype(np.uint16)
    pcm[:, :2000] = 2048 + rng.integers(-3, 4, (B, 2000))
    seg = np.stack([rng.integers(1, 3000, B), rng.integers(4000, U + 1, B)], 1).astype(np.uint32)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    atap["mid_val"] = 2048
    want = po.mfcc_geom_b_batch(pcm, seg, atap) if i %% 2 else po.mfcc_batch(pcm, seg, atap)
    case.append((pcm, seg, atap, want))
sr_b200.lib()                                     # loaded, nothing called yet: no CUDA context, no tables
bar = threading.Barrier(N, timeout=120)
res = [None] * N
def work(i):
    try:
        bar.wait()
        h = sr_b200.Handle(0)                     # 8 first uses at once: the per-device table upload
        pcm, seg, atap, want = case[i]
        if i %% 2:
            h.set_geometry(1)
        got = h.mfcc(pcm, seg, atap)
        res[i] = bool(ob.ftr_equal(got, want) and (got["frm_num"] > 0).all())
        h.close()
    except Exception as e:
        res[i] = repr(e)
ts = [threading.Thread(target=work, args=(i,)) for i in range(N)]
for t in ts: t.start()
for t in ts: t.join()
print("startup", res)
sys.exit(0 if all(r is True for r in res) else 1)
"""


@pytest.mark.gpu
def test_first_use_from_eight_threads_at_once():
    """a fresh process whose first library call is 8 sr_create at the same instant (the per-device MFCC tables are
    uploaded once, under a lock): every thread's get_mfcc batch, in both geometries, equals the oracle"""
    code = _STARTUP % (os.path.join(ROOT, "stm32-speech-recognition_b200", "python"), HERE)
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "startup [True, True, True, True, True, True, True, True]" in r.stdout, r.stdout[-3000:]
