"""Fixed captures at a rate (sr_streams_create_at_rate, include/sr_synth.h): per-push latency of the capture pool fed audio
at 16, 44.1 and 48 kHz, beside the 8 kHz pool fed the same audio resampled beforehand.

BASELINE configs[4]'s shape: 8 192 streams of 5 s captures (40 000 samples at 8 kHz), the 12-slot bank and the greedy
matcher. Stream s plays recording s % 64 of a set of distinct recordings, taken up to the rate by scipy's polyphase
filter; capture k of a run plays its seconds [5k, 5k + 5). For each rate and each chunk length (10 ms and 80 ms at the
rate) two setups alternate, twice each:
  * the pool at the rate, fed lock-step chunks at the rate from one pinned host buffer. A capture takes the pushes that
    complete its 40 000 8 kHz samples, one more than 5 s / chunk, because the last ~2 ms of input complete no output
    until more arrives;
  * the 8 kHz pool fed the recordings resampled beforehand by sr_resample_adc12_dev, in chunks of 80 / 640 samples.
Both pools are reset at every capture. For each run:
  * push p50 / p99: a host clock around the push, which returns after its one synchronisation;
  * kernel time per push: the CUDA kernels of 20 further pushes of the same setup under torch.profiler, in a pass of
    its own, in total and for stream_resample_kernel;
  * the check (at-rate runs): the events of 128 sampled streams equal those of the 8 kHz pool handed, at every push,
    the outputs [n8(before), n8(after)) of sr_resample_adc12_dev on the audio the stream was fed.
The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_stream_rate.py [--streams 8192] [--captures 2] [--rates 16000,44100,48000] [--json FILE]
"""
import argparse
import json
import time

import numpy as np
from scipy.signal import resample_poly

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import card, cuda_device, report
import oracle_bind as ob
import oracle_ext as ox
import resample_ref as rr
import sr_b200
import torch

NREC = 64
CAP = 40000                                     # 5 s captures at 8 kHz
REC_KEYS = ("stream", "segment", "start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")


def n8(n, rate):
    """the 8 kHz samples a stream at `rate` has after n input samples (include/sr_synth.h)"""
    L, M = rr.ratio(rate)
    c = (len(rr.taps(rate)) - 1) // 2
    return max(0, -(-(n * L - c) // M))


def pushes_per_capture(rate, c):
    """lock-step pushes of c input samples until a stream's 8 kHz stream holds CAP samples"""
    k = 1
    while n8(k * c, rate) < CAP:
        k += 1
    return k


def resample_dev(pcm, rate):
    """sr_resample_adc12_dev on the rows of pcm [B, U] at `rate`: [B, ceil(U L / M)] codes at 8 kHz"""
    B, U = pcm.shape
    U_out = rr.out_len(U, rate)
    x = torch.from_numpy(np.ascontiguousarray(pcm).view(np.int16)).cuda()
    out = torch.zeros((B, U_out), dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream()
    sr_b200.resample_adc12_dev(x.data_ptr(), U, B, None, rate, out.data_ptr(), U_out, None, st.cuda_stream)
    st.synchronize()
    return out.cpu().numpy().view(np.uint16)


def pcts(x):
    x = np.asarray(x) * 1e3
    return dict(p50_ms=float(np.percentile(x, 50)), p99_ms=float(np.percentile(x, 99)), mean_ms=float(x.mean()))


def kernel_ms(push, n):
    """CUDA kernel time of n calls of push() under torch.profiler: (total ms per push, stream_resample_kernel ms per push)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            push()
    total = rs = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = getattr(e, "cuda_time_total", 0.0) if t is None else t
        if "memcpy" in e.key.lower() or "memset" in e.key.lower():
            continue
        total += t
        if "stream_resample_kernel" in e.key:
            rs += t
    return total / 1e3 / n, rs / 1e3 / n


def run(h, recs, S, c, per_cap, captures, buf, ptr, rate=None, check=None):
    """rate None: the 8 kHz pool fed recs in chunks of c; else the pool at `rate` fed recs at that rate. Returns the row
    and, with check, the events of the sampled streams"""
    pool = sr_b200.StreamPool(h, S, CAP, 2400) if rate is None else sr_b200.StreamPool(h, S, CAP, 2400, rate=rate)
    rows = np.arange(S) % NREC
    view = buf[:S * c].reshape(S, c)
    sec = rate or 8000
    lat, events = [], 0
    got = {s: [] for s in (check or [])}
    for k in range(captures):
        pool.reset()
        base = 5 * sec * k
        for i in range(per_cap):
            view[:] = recs[:, base + i * c:base + (i + 1) * c][rows]
            t0 = time.perf_counter()
            ne = pool.push_raw(ptr, c, c)
            lat.append(time.perf_counter() - t0)
            events += ne
            for j in range(ne):
                e = pool._ev[j]
                if e.stream in got:
                    got[e.stream].append(tuple(int(getattr(e, f)) for f in REC_KEYS) + (k,))
    pool.reset()
    view[:] = recs[:, :c][rows]
    ker, ker_rs = kernel_ms(lambda: pool.push_raw(ptr, c, c), 20)
    pool.close()
    wall = sum(lat)
    row = dict(pool="sr_streams at %d Hz" % rate if rate else "sr_streams (8 kHz, resampled beforehand)", rate=rate or 8000,
               chunk_samples=c, pushes=len(lat), **pcts(lat), kernel_ms_per_push=ker, resample_kernel_ms_per_push=ker_rs,
               stream_seconds_per_second=S * len(lat) * c / sec / wall, events=events)
    return row, got


def oracle(h, recs_r, check, c, per_cap, captures, rate):
    """the 8 kHz pool on the sampled streams, handed at every push the outputs [n8(before), n8(after)) of
    sr_resample_adc12_dev on the audio each stream was fed"""
    S = len(check)
    pool = sr_b200.StreamPool(h, S, CAP, 2400)
    rows = np.asarray(check) % NREC
    want = {s: [] for s in check}
    for k in range(captures):
        pool.reset()
        base = 5 * rate * k
        audio = recs_r[rows, base:base + per_cap * c]
        eight = resample_dev(audio, rate)
        for i in range(per_cap):
            a, b = n8(i * c, rate), n8((i + 1) * c, rate)
            ch = np.ascontiguousarray(eight[:, a:b]) if b > a else np.zeros((S, 1), np.uint16)
            for e in pool.push_ragged(ch, np.full(S, b - a, np.uint32)):
                want[check[e["stream"]]].append(tuple(int(e[f]) if f != "stream" else check[e["stream"]]
                                                      for f in REC_KEYS) + (k,))
    pool.close()
    return want


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--captures", type=int, default=2, help="5 s captures per run")
    ap.add_argument("--rates", default="16000,44100,48000")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    rates = [int(r) for r in args.rates.split(",")]
    if any(r not in sr_b200.RESAMPLE_RATES or r == 8000 for r in rates):
        ap.error("--rates: rates of %s other than 8000" % (sr_b200.RESAMPLE_RATES,))
    cuda_device("bench_stream_rate")
    S = args.streams
    recs = ox.synth_long(NREC, 8000 * (5 * args.captures + 1), 0x5EED1500)
    tpl = sr_b200.synth_pcm_host(12, 8000, 0x7E3A0000)
    bank = sr_b200.make_bank(ob.port().recognise_batch(tpl, 2400, None, 0, 4096)["ftr"])
    h = sr_b200.Handle(0)
    h.set_bank(bank, 12, 4096)
    check = sorted(set(np.linspace(0, S - 1, 128).astype(int).tolist()))
    out_rows, ok = [], True
    arr, ptr = sr_b200.host_alloc_dev(0, S * (max(rates) // 100 * 8) * 2)
    buf = arr.view(np.uint16)
    try:
        for rate in rates:
            L, M = rr.ratio(rate)
            up = resample_poly(recs.astype(np.float64) - 2048, M, L, axis=1)
            recs_r = np.clip(np.rint(up + 2048), 0, 4095).astype(np.uint16)
            recs_8 = np.ascontiguousarray(resample_dev(recs_r, rate))
            for c in (rate // 100, rate // 100 * 8):
                c8 = c * L // M
                per_cap = pushes_per_capture(rate, c)
                for rep in range(2):
                    row, got = run(h, recs_r, S, c, per_cap, args.captures, buf, ptr, rate=rate,
                                   check=check if rep == 0 else None)
                    if rep == 0:
                        want = oracle(h, recs_r, check, c, per_cap, args.captures, rate)
                        same = all(sorted(got[s]) == sorted(want[s]) for s in check)
                        ok &= same
                        row.update(checked_streams=len(check), checked_events=sum(len(v) for v in want.values()),
                                   oracle_equal=same)
                    out_rows.append(row)
                    print(json.dumps(row), flush=True)
                    row, _ = run(h, recs_8, S, c8, CAP // c8, args.captures, buf, ptr)
                    out_rows.append(row)
                    print(json.dumps(row), flush=True)
    finally:
        h.close()
        sr_b200.host_free(ptr)
    print("%-9s %-14s %-44s %-22s %s" % ("rate", "chunk", "pool", "p50 / p99 ms", "kernels / resample ms per push"))
    for r in out_rows:
        print("%-9d %-14s %-44s %-22s %.3f / %.3f" % (r["rate"], r["chunk_samples"], r["pool"],
                                                      "%.3f / %.3f" % (r["p50_ms"], r["p99_ms"]),
                                                      r["kernel_ms_per_push"], r["resample_kernel_ms_per_push"]))
    report("bench_stream_rate", dict(card=card(), streams=S, captures=args.captures, rows=out_rows), ok, args.json)


if __name__ == "__main__":
    main()
