"""The standard ways the tests call the library on a GPU (TEST INFRASTRUCTURE): a handle with a bank and a matcher, the
timing tags, the device forms of recognition on torch buffers read back as the host calls return them, stream pushes and
their events checked against the oracles, and the comparisons of recognition records. torch is imported inside the
functions, so that CPU-only runs never import it. Bare asserts here are not rewritten by pytest, so each one carries a
message."""
import numpy as np

import lifter_ref
import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from refs import decide

NULL = 0xFFFFFFFF
LONG_REC = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


# ---- handles ---------------------------------------------------------------------------------------------------------
def handle(bank, T, flags=0, r=0):
    """a handle on device 0 with bank (T slots of 4 096 bytes) and the matcher (flags, r)"""
    h = sr_b200.Handle(0)
    h.set_bank(bank, T, 4096)
    h.set_match(flags, r)
    return h


def tags(h):
    """the timing tags collected since the last collect, in launch order"""
    return [t for t, _ in h.timing_collect()]


def tag_counts(h):
    """{tag: launches} collected since the last collect"""
    t = tags(h)
    return {k: t.count(k) for k in set(t)}


def enrolled_bank(h, n_cmd, seed):
    """one enrolled word per command at slot 4 * cmd (the other slots erased), from synthetic one-word captures"""
    pcm = sr_b200.synth_pcm_host(n_cmd, 8000, seed)
    enr, st = h.enrol(pcm, 2400)
    bank = np.full((4 * n_cmd, 4096), 0xFF, np.uint8)
    bank[::4] = enr
    return bank, pcm, st


def prefilled(h, pcm, P, max_words, n_len):
    """sr_recognise_connected_batch outputs for pcm's rows, every byte 0x5A"""
    shape = h.recognise_connected(pcm[:1], P, max_words, n_len)
    out = {k: np.frombuffer(b"\x5a" * a.nbytes, a.dtype).reshape(a.shape).copy() for k, a in shape.items()}
    return {k: np.repeat(v, pcm.shape[0], axis=0) for k, v in out.items()}


# ---- the device forms on torch buffers -------------------------------------------------------------------------------
def recognise_dev_launch(h, pcm, n_len, T, fields=sr_b200.RECOG_FIELDS, gather=()):
    """one sr_recognise_batch_dev launch of pcm [B, U] on the handle's stream, which must be the current torch stream,
    into fresh torch buffers prefilled with 0x5A / 0xA5 bytes for the fields named in `fields` (the others NULL). gather
    names the gathered outputs of a world of one rank ("score": [B][T] u32, "best": [B] u64 keys): then the call is
    sr_recognise_batch_dev_allgather, into buffers of their own. Returns the buffers, nothing synchronised"""
    import torch
    dev = torch.device("cuda:0")
    B, U = pcm.shape
    out = {"pcm": torch.from_numpy(pcm.view(np.int16)).to(dev)}
    full = {"atap": (B * 12, 0xA5, torch.uint8), "seg_off": (B * 6, 0x5A5A5A5A, torch.int32),
            "ftr": (B * sr_b200.FTR_BYTES, 0x5A, torch.uint8), "score": (B * max(T, 1), 0x5A5A5A5A, torch.int32),
            "status": (B, 0x5A, torch.uint8), "best_idx": (B, 0x5A5A5A5A, torch.int32),
            "best_dis": (B, 0x5A5A5A5A, torch.int32), "cmd": (B, 0x5A5A5A5A, torch.int32),
            "gathered_score": (B * max(T, 1), 0x5A5A5A5A, torch.int32), "gathered_best": (B, 0x5A5A5A5A5A5A5A5A, torch.int64)}
    for key in list(fields) + ["gathered_" + g for g in gather]:
        n, fill, dt = full[key]
        out[key] = torch.full((n,), fill, dtype=dt, device=dev)
    ptrs = {key: out[key].data_ptr() for key in fields}
    if gather:
        gs, gb = (out["gathered_" + g].data_ptr() if g in gather else None for g in ("score", "best"))
        h.recognise_dev_allgather(out["pcm"].data_ptr(), U, B, n_len, gathered_score=gs, gathered_best=gb, **ptrs)
    else:
        h.recognise_dev(out["pcm"].data_ptr(), U, B, n_len, **ptrs)
    return dict(out, B=B, T=T)


def recognise_dev_read(bufs):
    """the buffers of recognise_dev_launch, once their work is done, as the host call returns the fields (gathered_score
    [B, T] u32, gathered_best [B] u64)"""
    B, T = bufs["B"], bufs["T"]
    got = {key: v.cpu().numpy() for key, v in bufs.items() if key not in ("B", "T", "pcm")}
    if "atap" in got:
        got["atap"] = got["atap"].view(sr_b200.ATAP_DTYPE)
    if "ftr" in got:
        got["ftr"] = got["ftr"].view(sr_b200.FTR_DTYPE)
    if "seg_off" in got:
        got["seg_off"] = got["seg_off"].view(np.uint32).reshape(B, 3, 2)
    for key in ("score", "gathered_score"):
        if key in got:
            got[key] = got[key].view(np.uint32).reshape(B, -1)[:, :T]
    for key in ("best_idx", "best_dis", "cmd"):
        if key in got:
            got[key] = got[key].view(np.uint32)
    if "gathered_best" in got:
        got["gathered_best"] = got["gathered_best"].view(np.uint64)
    return got


def recognise_dev_np(h, pcm, n_len, T):
    """one sr_recognise_batch_dev launch on the whole batch; every output field, as the host call returns it"""
    import torch
    st = torch.cuda.Stream(torch.device("cuda:0"))
    h.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        bufs = recognise_dev_launch(h, pcm, n_len, T)
    st.synchronize()
    return recognise_dev_read(bufs)


def recognise_long_dev_np(h, pcm, lens, max_segs):
    """one sr_recognise_long_batch_dev call (n_len 2 400) on torch buffers: dict(n_segs, segs) as the host call returns
    them"""
    import torch
    dev = torch.device("cuda:0")
    B, U = pcm.shape
    d_pcm = torch.from_numpy(pcm.view(np.int16)).to(dev)
    d_lens = torch.from_numpy(lens.view(np.int32)).to(dev)
    d_n = torch.zeros(B, dtype=torch.int32, device=dev)
    d_segs = torch.zeros(B * max_segs * 7, dtype=torch.int32, device=dev)
    h.recognise_long_batch_dev(d_pcm.data_ptr(), U, B, d_lens.data_ptr(), 2400, max_segs, None, d_n.data_ptr(),
                               d_segs.data_ptr())
    h.sync()
    return dict(n_segs=d_n.cpu().numpy().view(np.uint32),
                segs=d_segs.cpu().numpy().view(ox.LONG_SEG_DTYPE).reshape(B, max_segs))


# ---- comparisons -----------------------------------------------------------------------------------------------------
def same(got, want, what):
    """a recognition result equals the oracle's composition, field by field"""
    for k in ("seg_off", "score", "best_idx", "best_dis", "cmd", "status"):
        g, w = np.asarray(got[k]).reshape(len(want["status"]), -1), want[k].reshape(len(want["status"]), -1)
        bad = np.flatnonzero((g != w).any(axis=1))
        assert len(bad) == 0, (what, k, bad[:8].tolist())
    assert ob.ftr_equal(got["ftr"], want["ftr"]), what


def cmp_long(got, want):
    """sr_recognise_long_batch records: n_segs and every record up to it"""
    for b in range(len(want["n_segs"])):
        assert got["n_segs"][b] == want["n_segs"][b], b
        m = min(int(want["n_segs"][b]), got["segs"].shape[1])
        assert got["segs"][b, :m].tobytes() == want["segs"][b, :m].tobytes(), (b, got["segs"][b, :m], want["segs"][b, :m])


def cmp_long_atap(got, want, rows=None):
    """cmp_long on the recordings of rows (default all), and each one's atap"""
    rows = range(len(want["n_segs"])) if rows is None else rows
    for b in rows:
        assert got["n_segs"][b] == want["n_segs"][b], b
        assert got["atap"][b].tobytes() == want["atap"][b].tobytes(), b
        m = min(int(want["n_segs"][b]), got["segs"].shape[1])
        assert got["segs"][b, :m].tobytes() == want["segs"][b, :m].tobytes(), (b, got["segs"][b, :m], want["segs"][b, :m])


# ---- streams ---------------------------------------------------------------------------------------------------------
def event_key(e):
    """(stream, segment) of a stream event"""
    return (int(e["stream"]), int(e["segment"]))


def k4_events(pool, pcm, arrival, rng, on_push=None):
    """fixed-capture pushes of pcm, "lockstep" (800 samples each) or ragged: (events, on_push(p) of the push that returned
    each); on_push(p) runs before push p"""
    S, L = pcm.shape
    events, pos, p = [], np.zeros(S, np.int64), 0
    while (pos < L).any():
        m = on_push(p) if on_push else None
        if arrival == "lockstep":
            lens = np.full(S, min(800, L - int(pos[0])), np.int64)
        else:
            lens = np.minimum(rng.choice([0, 1, 79, 81, 160, 333, 1601, 4000], S), L - pos)
        w = int(lens.max())
        p += 1
        if w == 0:
            continue
        chunk = np.zeros((S, w), np.uint16)
        for s in range(S):
            chunk[s, :lens[s]] = pcm[s, pos[s]:pos[s] + lens[s]]
        evs = pool.push(chunk) if arrival == "lockstep" else pool.push_ragged(chunk, lens)
        events += [(e, m) for e in evs]
        pos += lens
    return events


def check_k4(events, pool, pcm, bank, T, matcher=None):
    """every closed segment has one event, and each equals the oracle's get_mfcc of its segment, then the scan under the
    matcher of its push (matcher when the pushes did not switch it) and its decision: a matcher (flags, r) decides by the
    first-wins argmin, (flags, r, k, q) by SR_DTW_KNN(k) | SR_DTW_REJECT(q) (refs.decide); flags may hold SR_DTW_LIFTER"""
    ora = ob.best_oracle()
    seg, atap = pool.segments()
    S = pcm.shape[0]
    closed = [(s, k) for s in range(S) for k in range(3) if seg[s, k, 1] != NULL]
    got = sorted((e["stream"], e["segment"]) for e, _ in events)
    assert got == closed and len(closed) >= 2 * S, (got[:8], closed[:8], len(got), len(closed), S)
    for e, m in events:
        m = m if m is not None else matcher
        flags, r = m[:2]
        s, k = e["stream"], e["segment"]
        f = ora.mfcc_batch(pcm[s:s + 1], seg[s, k].reshape(1, 2), atap[s:s + 1])
        assert e["frm_num"] == int(f["frm_num"][0]), e
        if e["frm_num"] == 0:
            assert (e["status"], e["best_idx"], e["best_dis"]) == (2, 0, NULL), e
            continue
        idx, dis, cmd, rej = decide(lifter_ref.match_scores(f, bank, T, flags, r), *m[2:])
        want = (3 if rej[0] else 0, int(idx[0]), int(dis[0]), int(cmd[0]))
        assert (e["status"], e["best_idx"], e["best_dis"], e["cmd"]) == want, (m, e)


def k14_events(pool, xs, c, on_push=None):
    """lock-step pushes of c samples (shorter streams get 0 once done), then the queue drained: (event, matcher) pairs"""
    S, out, n, p = len(xs), [], np.zeros(len(xs), np.int64), 0
    N = np.array([len(x) for x in xs])
    while (n < N).any():
        m = on_push(p) if on_push else None
        lens = np.minimum(c, N - n)
        chunk = np.zeros((S, max(1, int(lens.max()))), np.uint16)
        for s in range(S):
            chunk[s, :lens[s]] = xs[s][n[s]:n[s] + lens[s]]
        out += [(e, m) for e in pool.push_ragged(chunk, lens.astype(np.uint32))]
        n += lens
        p += 1
    pending = pool.pending()
    assert pending == 0, pending                       # every event came out with the push that decided it
    return out


def long_records(pcm, lens, bank, T, m, max_segs=256):
    """the composed oracle's sr_recognise_long_batch records of pcm under the matcher m: (flags, r), or (flags, r, k, q)
    with SR_DTW_KNN(k) | SR_DTW_REJECT(q); flags may hold SR_DTW_LIFTER"""
    w = lifter_ref.recognise_long(ox.long_oracle(), ob.port(), pcm, 2400, bank, T, 4096, max_segs, lens, match=m[:2])
    if len(m) == 2:
        return w
    return ox.long_under_rule(w, pcm, 2400, lens, bank, T, m[:2], *m[2:], scores=lifter_ref.match_scores)


def check_k14(events, xs, bank, T, matchers):
    """each event equals the composed oracle's record of its whole recording under the matcher of its push (matchers[0]
    when the pushes did not switch it; a matcher as long_records takes it), in segment order, and every closed segment is
    handed out once"""
    S = len(xs)
    Ul = max(len(x) for x in xs)
    pcm = np.zeros((S, Ul), np.uint16)
    lens = np.array([len(x) for x in xs], np.uint32)
    for s, x in enumerate(xs):
        pcm[s, :len(x)] = x
    want = {m: long_records(pcm, lens, bank, T, m) for m in matchers}
    per = [0] * S
    for e, m in events:
        m = m if m is not None else matchers[0]                 # pushes without a switch: the pool's one matcher
        s, k = e["stream"], e["segment"]
        assert k == per[s], (s, k, per[s])
        per[s] += 1
        rec = want[m]["segs"][s, k]
        assert tuple(int(e[q]) for q in LONG_REC) == tuple(int(rec[q]) for q in LONG_REC), (m, e, rec)
    w = want[matchers[0]]
    for s in range(S):
        closed = [k for k in range(int(w["n_segs"][s])) if w["segs"][s, k]["status"] != 1]
        assert per[s] == len(closed), s
    assert sum(per) > 3 * S, per
