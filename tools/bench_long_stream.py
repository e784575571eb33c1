"""Live streams of any length (include/sr_long_stream.h): per-push latency and sustained real-time capacity.

8 192 streams of synthetic speech (many words each) are pushed in 10 ms and 80 ms chunks for --seconds of audio (60 by
default) from one pinned host buffer, so the step kernel reads each chunk in place. Stream s plays recording s % 64 of a
set of distinct recordings, started (s // 64) % 30 seconds into it. For each chunk length:
  * per-push latency p50 / p99: a host clock around sr_long_streams_push, which returns after its one synchronisation;
  * real-time capacity: stream-seconds of audio per wall second of pushing, and events per second;
  * the same for sr_streams_* (the fixed-capture pool) on 5 s streams, reset every 5 s;
  * the check: the events of 128 sampled streams equal the closed records of sr_recognise_long_batch on the audio they
    were fed.
The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_long_stream.py [--streams 8192] [--seconds 60] [--json FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "stm32-speech-recognition_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import oracle_bind as ob  # noqa: E402
import oracle_ext as ox  # noqa: E402
import sr_b200  # noqa: E402
from bench_match import card  # noqa: E402

NREC = 64
REC_KEYS = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


def stream_audio(recs, s, total):
    """the audio stream s plays: recording s % NREC from (s // NREC) % 30 seconds in, wrapping"""
    r = recs[s % NREC]
    off = 8000 * ((s // NREC) % 30)
    idx = (off + np.arange(total)) % len(r)
    return r[idx]


def pcts(x):
    x = np.asarray(x) * 1e3
    return dict(p50_ms=float(np.percentile(x, 50)), p99_ms=float(np.percentile(x, 99)), mean_ms=float(x.mean()))


def run_long(h, recs, S, c, total, buf, ptr, check):
    pool = sr_b200.LongStreamPool(h, S, c, 2400)
    evbuf = (sr_b200.StreamEvent * pool.max_events)()
    rows = np.arange(S) % NREC
    offs = 8000 * ((np.arange(S) // NREC) % 30)
    L = recs.shape[1]
    lat, events, got = [], 0, {s: [] for s in check}
    view = buf[:S * c].reshape(S, c)
    for n in range(0, total, c):
        view[:] = recs[rows[:, None], (offs[:, None] + n + np.arange(c)[None, :]) % L]
        t0 = time.perf_counter()
        ne = pool.push(ptr, c, c, events=evbuf)
        lat.append(time.perf_counter() - t0)
        events += ne
        for i in range(ne):
            e = evbuf[i]
            if e.stream in got:
                assert e.segment == len(got[e.stream])
                got[e.stream].append(tuple(getattr(e, k) for k in REC_KEYS))
    assert pool.pending() == 0
    pool.close()
    # the check: sr_recognise_long_batch on the audio each sampled stream was fed
    pcm = np.stack([stream_audio(recs, s, total) for s in check])
    r = h.recognise_long_batch(pcm, total // (19 * 80) + 4, 2400)
    for i, s in enumerate(check):
        recs_s = [tuple(int(v) for v in x) for x in r["segs"][i, :int(r["n_segs"][i])].tolist()]
        assert got[s] == [t for t in recs_s if t[2] != 1], s
    wall = sum(lat)
    return dict(pool="sr_long_streams", chunk_samples=c, pushes=len(lat), **pcts(lat),
                stream_seconds_per_second=S * total / 8000 / wall, events=events, events_per_second=events / wall,
                checked_streams=len(check), checked_events=sum(len(v) for v in got.values()))


def run_fixed(h, recs, S, c, total, buf, ptr):
    cap = 40000                                       # 5 s captures
    pool = sr_b200.StreamPool(h, S, cap, 2400)
    rows = np.arange(S) % NREC
    offs = 8000 * ((np.arange(S) // NREC) % 30)
    L = recs.shape[1]
    lat, events = [], 0
    view = buf[:S * c].reshape(S, c)
    for n0 in range(0, total, cap):
        pool.reset()
        for n in range(n0, min(n0 + cap, total), c):
            k = min(c, n0 + cap - n)
            view[:, :k] = recs[rows[:, None], (offs[:, None] + n + np.arange(k)[None, :]) % L]
            t0 = time.perf_counter()
            ne = pool.push_raw(ptr, k, c)
            lat.append(time.perf_counter() - t0)
            events += ne
    pool.close()
    wall = sum(lat)
    return dict(pool="sr_streams (5 s captures)", chunk_samples=c, pushes=len(lat), **pcts(lat),
                stream_seconds_per_second=S * total / 8000 / wall, events=events, events_per_second=events / wall)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--chunks", default="80,640", help="chunk lengths in samples (10 ms, 80 ms)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_stream: no CUDA device (there is nothing to measure without one)")
    S, total = args.streams, 8000 * args.seconds
    recs = ox.synth_long(NREC, 8000 * 60, 0x5EED1400)
    tpl = sr_b200.synth_pcm_host(12, 8000, 0x7E3A0000)
    bank = sr_b200.make_bank(ob.port().recognise_batch(tpl, 2400, None, 0, 4096)["ftr"])
    h = sr_b200.Handle(0)
    h.set_bank(bank, 12, 4096)
    chunks = [int(c) for c in args.chunks.split(",")]
    nbytes = S * max(chunks) * 2
    arr, ptr = sr_b200.host_alloc_dev(0, nbytes)
    buf = arr.view(np.uint16)
    check = sorted(set(np.linspace(0, S - 1, 128).astype(int).tolist()))
    rows = []
    try:
        for c in chunks:
            rows.append(run_long(h, recs, S, c, total, buf, ptr, check))
            print(json.dumps(rows[-1]), flush=True)
            rows.append(run_fixed(h, recs, S, c, total, buf, ptr))
            print(json.dumps(rows[-1]), flush=True)
    finally:
        h.close()
        sr_b200.host_free(ptr)
    res = dict(card=card(), streams=S, seconds=args.seconds, rows=rows)
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
