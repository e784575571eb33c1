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

With --rate (a rate of sr_b200.RESAMPLE_RATES other than 8000), the recordings are taken up to that rate first (scipy's
polyphase filter), and for each chunk length -- 10 ms and 80 ms at the rate -- two setups alternate, twice each:
  * the pool at the rate (sr_long_streams_create_at_rate) fed the chunks at the rate, which it resamples on the GPU;
  * the 8 kHz pool fed the same recordings resampled beforehand by sr_resample_adc12_dev, in 10 ms / 80 ms chunks.
Both report push p50 / p99 as above; the check compares the at-rate pool's sampled streams with sr_resample_adc12_dev on
the audio they were fed, followed by sr_recognise_long_batch.

    python tools/bench_long_stream.py [--streams 8192] [--seconds 60] [--rate 48000] [--json FILE]
"""
import argparse
import json
import time

import numpy as np

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import card, cuda_device, report
import oracle_bind as ob
import oracle_ext as ox
import sr_b200

NREC = 64
REC_KEYS = ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


def stream_audio(recs, s, total, rate=8000):
    """the audio stream s plays: recording s % NREC from (s // NREC) % 30 seconds in, wrapping"""
    r = recs[s % NREC]
    off = rate * ((s // NREC) % 30)
    idx = (off + np.arange(total)) % len(r)
    return r[idx]


def pcts(x):
    x = np.asarray(x) * 1e3
    return dict(p50_ms=float(np.percentile(x, 50)), p99_ms=float(np.percentile(x, 99)), mean_ms=float(x.mean()))


def resample_dev(pcm, rate):
    """sr_resample_adc12_dev on the rows of pcm [B, U] at `rate`: [B, ceil(U L / M)] codes at 8 kHz"""
    import torch
    B, U = pcm.shape
    U_out = -(-U * 8000 // rate)                      # ceil(U L / M) for (L, M) = (8000, rate) / gcd
    x = torch.from_numpy(np.ascontiguousarray(pcm).view(np.int16)).cuda()
    out = torch.zeros((B, U_out), dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U, B, None, rate, out.data_ptr(), U_out, None, st.cuda_stream)
    st.synchronize()
    return out.cpu().numpy().view(np.uint16)


def n8(n, rate):
    """the 8 kHz samples an at-rate stream has after n input samples (include/sr_synth.h)"""
    import resample_ref as rr
    L, M = rr.ratio(rate)
    c = (len(rr.taps(rate)) - 1) // 2
    return max(0, -(-(n * L - c) // M))


def run_long(h, recs, S, c, total, buf, ptr, check, rate=None):
    """rate None: the 8 kHz pool; else the pool at `rate`, fed recs at that rate (c and total count its samples)"""
    pool = sr_b200.LongStreamPool(h, S, c, 2400) if rate is None else sr_b200.LongStreamPool(h, S, c, 2400, rate=rate)
    evbuf = (sr_b200.StreamEvent * pool.max_events)()
    rows = np.arange(S) % NREC
    offs = (rate or 8000) * ((np.arange(S) // NREC) % 30)
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
    # the check: sr_recognise_long_batch on the audio each sampled stream was fed (at a rate: its first n8 outputs of
    # sr_resample_adc12_dev)
    pcm = np.stack([stream_audio(recs, s, total, rate or 8000) for s in check])
    if rate is not None:
        pcm = np.ascontiguousarray(resample_dev(pcm, rate)[:, :n8(total, rate)])
    r = h.recognise_long_batch(pcm, pcm.shape[1] // (19 * 80) + 4, 2400)
    for i, s in enumerate(check):
        recs_s = [tuple(int(v) for v in x) for x in r["segs"][i, :int(r["n_segs"][i])].tolist()]
        assert got[s] == [t for t in recs_s if t[2] != 1], s
    wall = sum(lat)
    row = dict(pool="sr_long_streams", chunk_samples=c, pushes=len(lat), **pcts(lat),
               stream_seconds_per_second=S * total / (rate or 8000) / wall, events=events, events_per_second=events / wall,
               checked_streams=len(check), checked_events=sum(len(v) for v in got.values()))
    if rate is not None:
        row.update(pool="sr_long_streams at %d Hz" % rate, rate=rate)
    return row


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


def main_rate(args, h, recs, S, check):
    """--rate: the at-rate pool against the 8 kHz pool fed the same recordings resampled beforehand, alternating"""
    from scipy.signal import resample_poly
    rate = args.rate
    g = np.gcd(8000, rate)
    up = np.clip(np.rint(resample_poly(recs.astype(np.float64) - 2048, rate // g, 8000 // g, axis=1) + 2048), 0, 4095)
    recs_r = up.astype(np.uint16)
    recs_8 = np.ascontiguousarray(resample_dev(recs_r, rate)[:, :recs.shape[1]])
    chunks = [rate // 100, rate // 100 * 8]
    arr, ptr = sr_b200.host_alloc_dev(0, S * max(chunks) * 2)
    buf = arr.view(np.uint16)
    rows = []
    try:
        for c in chunks:
            c8 = c * 8000 // rate
            for rep in range(2):
                rows.append(run_long(h, recs_r, S, c, rate * args.seconds, buf, ptr, check, rate=rate))
                print(json.dumps(rows[-1]), flush=True)
                rows.append(run_long(h, recs_8, S, c8, 8000 * args.seconds, buf, ptr, check))
                rows[-1].update(pool="sr_long_streams (8 kHz, resampled beforehand)")
                print(json.dumps(rows[-1]), flush=True)
    finally:
        sr_b200.host_free(ptr)
    return dict(card=card(), streams=S, seconds=args.seconds, rate=rate, rows=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--chunks", default="80,640", help="chunk lengths in samples (10 ms, 80 ms)")
    ap.add_argument("--rate", type=int, default=None, help="input rate of the at-rate pool (see above)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.rate is not None and (args.rate not in sr_b200.RESAMPLE_RATES or args.rate == 8000):
        ap.error("--rate: one of %s other than 8000" % (sr_b200.RESAMPLE_RATES,))
    cuda_device("bench_long_stream")
    S, total = args.streams, 8000 * args.seconds
    recs = ox.synth_long(NREC, 8000 * 60, 0x5EED1400)
    tpl = sr_b200.synth_pcm_host(12, 8000, 0x7E3A0000)
    bank = sr_b200.make_bank(ob.port().recognise_batch(tpl, 2400, None, 0, 4096)["ftr"])
    h = sr_b200.Handle(0)
    h.set_bank(bank, 12, 4096)
    if args.rate is not None:
        check = sorted(set(np.linspace(0, S - 1, 128).astype(int).tolist()))
        try:
            out = main_rate(args, h, recs, S, check)
        finally:
            h.close()
        report("bench_long_stream", out, True, args.json)
        return
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
    report("bench_long_stream", dict(card=card(), streams=S, seconds=args.seconds, rows=rows), True, args.json)


if __name__ == "__main__":
    main()
