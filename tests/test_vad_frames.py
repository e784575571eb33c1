"""The VAD frame by frame (csrc/sr_vad_core.cuh: block_scan, block_scan_split8, block_flags, frames_pass) on inputs where
every frame of a region decides the segments, through every VAD path.

VAD's only output is its segment list, and a frame's frm_sum / frm_zero reaches that list only when an error flips the
frame's activity and the flip completes or breaks a run of 8 active or 11 inactive frames. Random and recorded inputs
almost never do both. The inputs here (cases.critical_pcm) do it on purpose: runs of exactly 8 active frames, then exactly
11 inactive ones, each critical frame's deciding feature exactly at its threshold (active: one unit above, inactive: at
it). So a +-1 error in any critical frame's frm_sum or frm_zero changes the segments. The families: sums decide
(z_thl >= 159), crossings decide (s_thl out of reach), and mixed (the feature that does not decide sits exactly at its
threshold, which tests the `||` of VAD.C:164).

CPU: the per-frame reference (refs.vad_frames + vad_fsm) equals the oracle and the reference's own C on the extreme,
fuzz and threshold-corner inputs; every critical input realises its plan, every single flip changes the segments, and the
case sets hit every entry of the coverage table (cases.COVER_UNITS, COVER_PLACES).
GPU: sr_vad_batch (host and _dev, misaligned PCM, odd U, buf_len < U), the drop-in VAD(), seg_off of sr_recognise_batch
(planned noise windows), sr_vad_long_batch (host and _dev, ragged lens), K4 stream pools (lock-step and ragged pushes) and
K14 long streams, each against vad_fsm(vad_frames(...)). Each case runs once."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as ob
import sr_b200
from cases import (COVER_PLACES, COVER_UNITS, U32, Bands, critical_pcm, frame_cover, frames_of, noise_window,
                   vad_atap)
from refs import NULL, py_vad, seg_table, vad_active, vad_frames, vad_fsm

# (family, atap) of the capped calls: the band of real captures, z_thl 0 (one crossing decides), a wrapped b_thl with
# n_thl > 32 768 (the packed compare reads only b_thl's low 16 bits), a_thl = 0, a_thl > 0xFFFF, b_thl = 0
CONFIGS = (("zero", (2048, 100, 0, U32)), ("zero", (2048, 100, 5, U32)), ("zero", (100, 40000, 3, U32)),
           ("zero", (150, 200, 1, U32)), ("sum", (2048, 100, 159, 20000)), ("sum", (0, 0, 200, 80000)),
           ("sum", (60000, 8000, 65535, 400000)), ("mixz", (2048, 100, 2, 9600)), ("mixz", (2048, 100, 0, 8000)),
           ("mixs", (2048, 100, 2, 12000)), ("mixs", (1000, 1000, 0, 60000)), ("mixs", (60000, 8000, 0, 300000)))
NFR = 97                    # 98 blocks: the last pass of K0 and K11b has 2 blocks (the split8 tail)
N_K0 = 80 * NFR + 160
NOISE = ((2048, 100, 8800), (2048, 60, 5500), (1000, 200, 17600))     # mid, n_thl, s_thl of the planned noise windows
LONG_NFR = 19 * 111 + 1     # 2 110 frames: two 1 024-frame window edges, the last group closes at the last frame


def _groups(rng, nfr, n_groups, last):
    """first frames of n_groups groups (19 frames each, gaps of 0-6 frames), the last one closing at frame nfr - 1 when
    last, else anywhere"""
    gaps = rng.integers(0, min(7, (nfr - 1 - 19 * n_groups) // max(1, n_groups - 1) + 1), n_groups)
    span = 19 * n_groups + int(gaps[1:].sum())
    g0 = nfr - span if last else int(rng.integers(1, nfr - span + 1))
    out, g = [], g0
    for j in range(n_groups):
        g += int(gaps[j]) if j else 0
        out.append(g)
        g += 19
    return out


def k0_cases(seed=0x7AD0):
    """the capped calls' critical captures of N_K0 samples (NFR frames): two per config, one of them closing at the last
    frame"""
    rng = np.random.default_rng(seed)
    out = []
    for i, (fam, at) in enumerate(CONFIGS):
        for last in (False, True):
            atap = vad_atap(*at)
            g = _groups(rng, NFR, 3, last)
            pcm, act, crit = critical_pcm(rng, atap, fam, NFR, g)
            out.append(dict(name="%s%d%s" % (fam, i, "L" if last else ""), family=fam, atap=atap, pcm=pcm, act=act,
                            crit=crit, cap=3))
    return out


def noise_cases(n_rows, nfr, seed, groups_per_row=3):
    """critical captures that start with a planned 2 400-sample noise window (noise_atap gives the atap, z_thl 2)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_rows):
        mid, n_thl, s_thl = NOISE[i % len(NOISE)]
        fam = ("zero", "mixs", "mixz")[i % 3]
        win, atap = noise_window(mid, n_thl, s_thl)
        g = _groups(rng, nfr - 31, groups_per_row, i % 2 == 1)
        g = [x + 31 for x in g]
        pcm, act, crit = critical_pcm(rng, atap, fam, nfr, g, prefix=win, bsum=(0.4, 0.6), bare=range(32, nfr, 32))
        out.append(dict(name="noise%d" % i, family=fam, atap=atap, pcm=pcm, act=act, crit=crit, cap=3))
    return out


def long_cases(seed=0x10AD):
    """long recordings critical from frame 0 to the last: back-to-back groups every 19 frames; ragged lengths"""
    rng = np.random.default_rng(seed)
    fams = (("zero", (2048, 100, 0, U32)), ("zero", (2048, 100, 5, U32)), ("zero", (100, 40000, 3, U32)),
            ("sum", (2048, 100, 159, 20000)), ("mixz", (2048, 100, 2, 9600)), ("mixs", (1000, 1000, 0, 60000)))
    out = []
    for i, (fam, at) in enumerate(fams):
        nfr = LONG_NFR - 19 * i
        atap = vad_atap(*at)
        pcm, act, crit = critical_pcm(rng, atap, fam, nfr, list(range(1, nfr - 18, 19)), n=80 * nfr + 81 + 13 * i)
        out.append(dict(name="long%d" % i, family=fam, atap=atap, pcm=pcm, act=act, crit=crit, cap=None))
    return out


_CACHE = {}


def case_set(which):
    if which not in _CACHE:
        _CACHE[which] = {"k0": k0_cases, "noise": lambda: noise_cases(9, NFR, 0x4015E),
                         "pool": lambda: noise_cases(12, NFR, 0x9001), "long": long_cases}[which]()
    return _CACHE[which]


def want_segs(c):
    return vad_fsm(c["act"], c["cap"])


# ---- CPU: the reference against the oracle ---------------------------------------------------------------------------
def _oracle_inputs():
    """the inputs of the existing VAD parity tests (extremes, fuzz with arbitrary atap, threshold corners), built the same
    way: [(pcm row, atap)]"""
    out = []
    rng = np.random.default_rng(4)
    pcm = sr_b200.synth_pcm_host(16, 8000, 0xABCD0000)
    pcm[0] = rng.integers(0, 4096, 8000)
    pcm[1] = rng.integers(0, 65536, 8000)
    pcm[2] = 2048
    pcm[3, 2400:] = np.where(np.arange(5600) % 2 == 0, 0, 4095)
    for b in range(5, 16):                                # sparse out-of-band spikes
        pcm[b] = 2048 + rng.integers(-3, 4, 8000)
        idx = rng.integers(2400, 8000, 60)
        pcm[b, idx] = np.where(rng.integers(0, 2, 60) == 1, 2048 + 500, 2048 - 500)
    po = ob.port()
    out += [(pcm[b], po.noise_atap(pcm[b], 2400)) for b in range(16)]
    rng = np.random.default_rng(77)
    for b in range(48):                                   # arbitrary atap, b_thl often wrapped
        kind = b % 4
        base = int(rng.integers(0, 4096))
        x = (rng.integers(0, 4096, 4000) if kind == 0 else rng.integers(0, 65536, 4000) if kind == 1 else
             np.where(rng.random(4000) < 0.05, rng.integers(0, 4096, 4000), base) if kind == 2 else
             np.where(rng.integers(0, 2, 51).repeat(80)[:4000] == 1, rng.integers(0, 4096, 4000), base))
        a = vad_atap(int(rng.integers(0, 4096)) if b >= 4 else int(rng.integers(60000, 2 ** 32, dtype=np.uint64)),
                     int(rng.integers(0, 3000)), int(rng.integers(0, 12)), int(rng.integers(0, 200000)))
        out.append((x.astype(np.uint16), a))
    rng = np.random.default_rng(2024)
    for mid, n in ((0, 0), (1, 1), (2048, 0), (2048, 2049), (65535, 0), (65000, 536), (65536, 1), (70000, 4465),
                   (2 ** 32 - 1, 1), (32768, 32768), (100, 40000)):
        c = min(mid, 65535)
        x = np.full(4000, c, np.int64)
        idx = rng.integers(0, 4000, 120)
        x[idx] = rng.choice([0, 65535, max(c - n, 0), min(c + n, 65535), max(c - n - 1, 0)], 120)
        out.append((x.astype(np.uint16), vad_atap(mid, n, int(rng.integers(0, 6)), int(rng.integers(0, 400000)))))
    return out


def test_reference_equals_oracle_and_reference_build():
    """vad_fsm(vad_frames(...)) is the oracle's VAD, and the reference's own VAD.C where it was built, on the extreme,
    fuzz and threshold-corner inputs of the parity tests and on the critical inputs here (capped at 3 segments)"""
    libs = [ob.port()] + ([ob.ref()] if ob.have_ref() else [])
    cases = [(x, a) for x, a in _oracle_inputs()] + [(c["pcm"], c["atap"]) for c in case_set("k0")]
    for i, (x, a) in enumerate(cases):
        want = seg_table(py_vad(x, len(x), a[0], 3)).reshape(-1).tolist()
        for lib in libs:
            assert lib.vad(x, len(x), a).tolist() == want, (i, type(lib).__name__)


def test_long_reference_equals_long_oracle():
    """uncapped, the pair is the long-form oracle (sro_vad_long_batch) on the long critical recordings, ragged lens"""
    import oracle_ext as ox
    cases = case_set("long")
    U = max(len(c["pcm"]) for c in cases)
    pcm = np.zeros((len(cases), U), np.uint16)
    for b, c in enumerate(cases):
        pcm[b, :len(c["pcm"])] = c["pcm"]
    atap = np.concatenate([c["atap"] for c in cases])
    n, seg = ox.long_oracle().vad_long(pcm, atap, 160, [len(c["pcm"]) for c in cases])
    for b, c in enumerate(cases):
        want = py_vad(c["pcm"], len(c["pcm"]), c["atap"][0])
        assert want == want_segs(c), c["name"]
        assert [tuple(t) for t in seg[b, :int(n[b])].tolist()] == want, c["name"]


# ---- CPU: the critical inputs are what they claim -------------------------------------------------------------------
@pytest.mark.parametrize("which", ["k0", "noise", "pool", "long"])
def test_critical_inputs_realise_their_plan(which):
    """every case: the reference's activity is the plan; each critical frame's deciding feature is one unit above (active)
    or exactly at (inactive) its threshold, the other feature at or under its own (exactly at it in the mixed families);
    flipping any single critical frame changes the segments"""
    for c in case_set(which):
        a0 = c["atap"][0]
        fr = vad_frames(c["pcm"], len(c["pcm"]), a0)
        act = vad_active(fr, a0)
        assert len(act) == len(c["act"]) == frames_of(len(c["pcm"])), c["name"]
        assert (act == c["act"]).all(), (c["name"], np.flatnonzero(act != c["act"])[:8])
        z, s = int(a0["z_thl"]), int(a0["s_thl"])
        k = np.flatnonzero(c["crit"])
        a = c["act"][k].astype(np.int64)
        fs, fz = fr[0][k], fr[1][k]
        fam = c["family"]
        if fam == "sum":
            assert (fs == s + a).all() and (fz <= z).all(), c["name"]
        elif fam == "zero":
            assert (fz == z + a).all() and (fs <= s).all(), c["name"]
        elif fam == "mixz":
            assert (fz == z + a).all() and (fs == s).all(), c["name"]
        else:
            assert (fs == s + a).all() and (fz == z).all(), c["name"]
        if which in ("noise", "pool"):                    # noise_atap over the planned window gives the planned atap
            assert ob.port().noise_atap(c["pcm"], 2400).tobytes() == c["atap"].tobytes(), c["name"]
        want = vad_fsm(c["act"], c["cap"])
        assert len(want) == (min(3, len(want)) if c["cap"] else (k.size - 1) // 19), c["name"]
        for j in k:
            flip = c["act"].copy()
            flip[j] = not flip[j]
            assert vad_fsm(flip, c["cap"]) != want, (c["name"], int(j))


def test_coverage_table_is_complete():
    """between them, the critical frames of the case sets hit every entry of the coverage table"""
    hit = {}
    for which in ("k0", "noise", "pool", "long"):
        for c in case_set(which):
            a0 = c["atap"][0]
            init = vad_frames(c["pcm"], len(c["pcm"]), a0)[2]
            nfr = len(c["act"])
            for k in np.flatnonzero(c["crit"]):
                for e in frame_cover(c["pcm"], c["atap"], int(k), int(init[k]), nfr, c["family"]):
                    hit[e] = hit.get(e, 0) + 1
    missing = [e for e in COVER_UNITS + COVER_PLACES if e not in hit]
    assert not missing, (missing, hit)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _rows(cases, U, buf_len=None):
    """[B, U] PCM of the cases (each case's samples, then poison up to U) and the atap array"""
    B = len(cases)
    pcm = np.zeros((B, U), np.uint16)
    atap = np.zeros(B, sr_b200.ATAP_DTYPE)
    for b, c in enumerate(cases):
        n = len(c["pcm"]) if buf_len is None else buf_len
        pcm[b, :n] = c["pcm"][:n]
        pcm[b, n:] = np.where(np.arange(U - n) % 2, 65535, 0)
        atap[b] = c["atap"][0]
    return pcm, atap


def _shifted(pcm, byte_off):
    """a copy of pcm whose first sample sits byte_off bytes past a 16-byte boundary"""
    raw = np.zeros(pcm.size * 2 + 64, np.uint8)
    base = (-raw.ctypes.data) % 16 + byte_off
    out = raw[base:base + pcm.size * 2].view(np.uint16).reshape(pcm.shape)
    out[:] = pcm
    assert out.ctypes.data % 16 == byte_off
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("byte_off", [0, 2, 6, 14])
def test_vad_batch_host(handle, byte_off):
    """sr_vad_batch on the critical captures, PCM 0, 2, 6 and 14 bytes past a 16-byte boundary"""
    cases = case_set("k0")
    pcm, atap = _rows(cases, N_K0)
    seg = handle.vad(_shifted(pcm, byte_off), atap)
    for b, c in enumerate(cases):
        assert seg[b].tolist() == seg_table(want_segs(c)).tolist(), (byte_off, c["name"])


@pytest.mark.gpu
@pytest.mark.parametrize("U,buf_len", [(N_K0 - 1, N_K0 - 1), (N_K0 + 333, N_K0)])
def test_vad_batch_odd_rows_and_short_buf_len(handle, U, buf_len):
    """odd U: rows start at odd sample shifts (every other row skips the split8 tail); buf_len < U: the rest of each row
    is poison. N_K0 - 1 samples still make NFR frames"""
    cases = case_set("k0")
    pcm, atap = _rows(cases, U, buf_len)
    seg = handle.vad(pcm, atap, buf_len)
    for b, c in enumerate(cases):
        want = py_vad(pcm[b], buf_len, atap[b], 3)
        assert want == want_segs(c), c["name"]
        assert seg[b].tolist() == seg_table(want).tolist(), (U, c["name"])


@pytest.mark.gpu
def test_vad_batch_dev(handle):
    """sr_vad_batch_dev on device PCM, outputs between sentinels"""
    import torch
    cases = case_set("k0")
    pcm, atap = _rows(cases, N_K0)
    B = len(cases)
    dev = torch.device("cuda:0")
    p = torch.from_numpy(pcm.view(np.int16)).to(dev)
    at = torch.from_numpy(atap.view(np.uint8).copy()).to(dev)
    sg = torch.full((B + 1, 6), 0x5A5A5A5A, dtype=torch.int32, device=dev)
    handle.vad_dev(p.data_ptr(), N_K0, B, N_K0, at.data_ptr(), sg.data_ptr())
    torch.cuda.synchronize()
    got = sg.cpu().numpy().view(np.uint32)
    assert (got[B] == 0x5A5A5A5A).all()
    for b, c in enumerate(cases):
        assert got[b].tolist() == seg_table(want_segs(c)).reshape(-1).tolist(), c["name"]


@pytest.mark.gpu
def test_drop_in_VAD(handle):
    """the reference-named VAD() on each critical capture: segment pointers into the caller's buffer"""
    L = sr_b200.lib()
    for c in case_set("k0"):
        pcm = np.ascontiguousarray(c["pcm"])
        vv = (sr_b200.ValidTag * 3)()
        L.VAD(pcm.ctypes.data_as(C.c_void_p), len(pcm), vv, c["atap"].ctypes.data_as(C.c_void_p))
        base = pcm.ctypes.data
        got = [((v.start - base) // 2 if v.start else NULL, (v.end - base) // 2 if v.end else NULL) for v in vv]
        assert [list(t) for t in got] == seg_table(want_segs(c)).tolist(), c["name"]


def _bank_handle():
    h = sr_b200.Handle(0)
    f = sr_b200.synth_ftr_host(4, 0xF7A3).view(sr_b200.FTR_DTYPE).reshape(-1)
    h.set_bank(sr_b200.make_bank(f), 4, 4096)
    return h


@pytest.mark.gpu
def test_recognise_seg_off_with_planned_noise_windows():
    """seg_off of sr_recognise_batch: noise_atap over the planned window gives the planned atap, then the critical frames"""
    cases = case_set("noise")
    pcm, _ = _rows(cases, N_K0)
    h = _bank_handle()
    try:
        out = h.recognise(pcm, 2400)
    finally:
        h.close()
    for b, c in enumerate(cases):
        assert out["atap"][b].tobytes() == c["atap"][0].tobytes(), c["name"]
        assert out["seg_off"][b].tolist() == seg_table(want_segs(c)).tolist(), c["name"]


def _long_rows(cases):
    U = max(len(c["pcm"]) for c in cases) + 7
    lens = np.array([len(c["pcm"]) for c in cases], np.uint32)
    pcm, atap = _rows(cases, U)
    for b, n in enumerate(lens):
        pcm[b, n:] = np.where(np.arange(U - n) % 3 == 0, 65535, 0)
    return pcm, atap, lens


@pytest.mark.gpu
def test_vad_long_host(handle):
    """sr_vad_long_batch with the caller's atap (n_len 0 keeps it), ragged lens: every segment of every recording"""
    cases = case_set("long")
    pcm, atap, lens = _long_rows(cases)
    M = 160
    v = handle.vad_long_batch(pcm, M, 0, lens, atap=atap.copy())
    for b, c in enumerate(cases):
        want = want_segs(c)
        assert int(v["n_segs"][b]) == len(want), c["name"]
        assert [tuple(t) for t in v["seg_off"][b, :len(want)].tolist()] == want, c["name"]


@pytest.mark.gpu
def test_vad_long_dev(handle):
    """sr_vad_long_batch_dev on device buffers, the same recordings"""
    import torch
    cases = case_set("long")
    pcm, atap, lens = _long_rows(cases)
    B, U = pcm.shape
    M = 160
    dev = torch.device("cuda:0")
    p = torch.from_numpy(pcm.view(np.int16)).to(dev)
    ln = torch.from_numpy(lens.view(np.int32)).to(dev)
    at = torch.from_numpy(atap.view(np.uint8).copy()).to(dev)
    ns = torch.zeros(B, dtype=torch.int32, device=dev)
    sg = torch.full((B, M, 2), 0x5A5A5A5A, dtype=torch.int32, device=dev)
    handle.vad_long_batch_dev(p.data_ptr(), U, B, ln.data_ptr(), 0, M, at.data_ptr(), ns.data_ptr(), sg.data_ptr())
    torch.cuda.synchronize()
    n_segs = ns.cpu().numpy()
    seg = sg.cpu().numpy().view(np.uint32)
    for b, c in enumerate(cases):
        want = want_segs(c)
        assert int(n_segs[b]) == len(want), c["name"]
        assert [tuple(t) for t in seg[b, :len(want)].tolist()] == want, c["name"]
        assert (seg[b, len(want):] == 0x5A5A5A5A).all(), c["name"]


def _carried_markers(c):
    """sample positions of the markers that a later critical frame carries in (the last marker before its block k)"""
    bd = Bands(c["atap"])
    cls = bd.cls(c["pcm"])
    mk = np.flatnonzero(cls)
    out = set()
    for k in np.flatnonzero(c["crit"]):
        before = mk[mk <= 80 * k + 78]
        if len(before) and before[-1] < 80 * k:
            out.add(int(before[-1]))
    return sorted(out)


def _push_plan(rng, c, max_chunk):
    """push boundaries at every residue mod 80 and just before and after each carried marker, chunks <= max_chunk"""
    n = len(c["pcm"])
    cuts = set(int(p) + d for p in _carried_markers(c) for d in (0, 1) if 0 < int(p) + d < n)
    pos = 0
    for r in rng.permutation(80):
        pos += 80 + int(r) if rng.random() < 0.5 else int(r) + 1
        if pos >= n:
            break
        cuts.add(pos)
    cuts = sorted(cuts | {n})
    lens, prev = [], 0
    for q in cuts:
        while q - prev > max_chunk:
            lens.append(max_chunk)
            prev += max_chunk
        if q > prev:
            lens.append(q - prev)
            prev = q
    return lens


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["lockstep", "ragged"])
def test_k4_pools(mode):
    """fixed-capture stream pools (K4): the planned noise window calibrates, the carried class crosses every push;
    lock-step chunks of 77 samples (every residue mod 80), or each stream's own plan"""
    cases = case_set("pool")
    S, L = len(cases), N_K0
    h = _bank_handle()
    pool = sr_b200.StreamPool(h, S, L, 2400)
    events = []
    try:
        if mode == "lockstep":
            for p0 in range(0, L, 77):
                chunk = np.stack([c["pcm"][p0:p0 + 77] for c in cases])
                events += pool.push(np.ascontiguousarray(chunk))
        else:
            rng = np.random.default_rng(0xC4)
            plans = [_push_plan(rng, c, 4000) for c in cases]
            at = np.zeros(S, np.int64)
            while any(plans):
                lens = np.array([p.pop(0) if p else 0 for p in plans], np.int64)
                chunk = np.zeros((S, max(1, int(lens.max()))), np.uint16)
                for s, c in enumerate(cases):
                    chunk[s, :lens[s]] = c["pcm"][at[s]:at[s] + lens[s]]
                events += pool.push_ragged(chunk, lens.astype(np.uint32))
                at += lens
        events += pool.fetch()
        seg, atap = pool.segments()
    finally:
        pool.close()
        h.close()
    got = {}
    for e in events:
        got.setdefault(e["stream"], []).append((e["segment"], e["start"], e["end"]))
    for s, c in enumerate(cases):
        want = want_segs(c)
        assert atap[s].tobytes() == c["atap"][0].tobytes(), c["name"]
        assert seg[s].tolist() == seg_table(want).tolist(), (mode, c["name"])
        closed = [(j, st, en) for j, (st, en) in enumerate(want) if en != NULL]
        assert sorted(got.get(s, [])) == closed, (mode, c["name"])


@pytest.mark.gpu
def test_k14_streams():
    """live streams of any length (K14) from the caller's atap: every segment handed out as it closes, the open one in
    the state, with push boundaries at every residue mod 80 and around each carried marker"""
    cases = case_set("long")
    S, max_chunk = len(cases), 3000
    atap0 = np.concatenate([c["atap"] for c in cases])
    h = _bank_handle()
    pool = sr_b200.LongStreamPool(h, S, max_chunk, 0, atap0)
    rng = np.random.default_rng(0x14)
    plans = [_push_plan(rng, c, max_chunk) for c in cases]
    got = [[] for _ in range(S)]
    at = np.zeros(S, np.int64)
    try:
        while any(plans):
            lens = np.array([p.pop(0) if p else 0 for p in plans], np.int64)
            chunk = np.zeros((S, max(1, int(lens.max()))), np.uint16)
            for s, c in enumerate(cases):
                chunk[s, :lens[s]] = c["pcm"][at[s]:at[s] + lens[s]]
            for e in pool.push_ragged(chunk, lens.astype(np.uint32)):
                got[e["stream"]].append((e["segment"], e["start"], e["end"]))
            at += lens
        for e in pool.fetch():
            got[e["stream"]].append((e["segment"], e["start"], e["end"]))
        st = pool.state()
    finally:
        pool.close()
        h.close()
    for s, c in enumerate(cases):
        want = want_segs(c)
        closed = [(j, a, b) for j, (a, b) in enumerate(want) if b != NULL]
        assert got[s] == closed, (c["name"], got[s][:3], closed[:3])
        op = want[-1][0] if want and want[-1][1] == NULL else NULL
        assert int(st["open_start"][s]) == op, c["name"]
