"""Throughput of the host-buffer capture calls at a rate (sr_recognise_batch_at_rate and sr_enrol_batch_at_rate,
include/sr_synth.h): 16 384 captures of 1 s at 16, 44.1 and 48 kHz in pinned host memory (1.57 GB at 48 kHz), against
bench.py's configs[1] bank (20 templates synthesised on the device). Recognition reads back seg_off, best_idx, best_dis,
cmd and status, as an application would; enrolment the bank image and status.

Per rate, alternating in one run, `--steps` calls of each (after `--warmup`):
  plain        sr_recognise_batch_at_rate with the transport forced plain: the input crosses PCIe as u16;
  packed       the same call with the transport forced packed (12 bits per sample where the host has CPUs to pack with);
  8k_fed       sr_recognise_batch on the same audio resampled beforehand (transport plain): the same kernels without K15
               and a sixth (48 kHz) of the bytes to copy;
  enrol        sr_enrol_batch_at_rate on the first `--enrol` captures;
  enrol_dev    the path it replaces: K15 on a device copy, the 8 kHz audio back to pinned memory, sr_enrol_batch.
Reported: wall ms per call (host clock around calls that end in a synchronisation), captures per second, the input bytes
the call copies host to device per second of the call (from sr_transport_stats for recognise), and tag 15's share of the
call (its kernel time over the call's wall time, from a separate timed window). Sampled captures are checked against the
CPU composition tests/resample_ref.py + the oracle port. The card's name, power limit and SM clock limit are read in the
same run.

    python tools/bench_capture_rate.py [--captures 16384] [--enrol 4096] [--steps 3] [--warmup 1] [--json FILE]
"""
import argparse
import json
import time

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import card, cuda_device, device_bank, per_call, report, timed
import oracle_bind as ob
import resample_ref as rr
import sr_b200

N_LEN = 2400
WANT = ("seg_off", "best_idx", "best_dis", "cmd", "status")     # what an application reads back


def pinned(shape):
    mem, ptr = sr_b200.host_alloc_dev(0, int(np.prod(shape)) * 2)
    return mem.view(np.uint16).reshape(shape), ptr


def captures_at(rate, B, seed):
    """B captures of 1 s: 64 distinct synthetic 8 kHz captures taken to `rate` by linear interpolation, repeated, pinned"""
    x8 = sr_b200.synth_pcm_host(64, 8000, seed, 3)
    out, ptr = pinned((B, rate))
    t = np.arange(rate) * (8000.0 / rate)
    base = np.stack([np.rint(np.interp(t, np.arange(8000), x8[b])).astype(np.uint16) for b in range(64)])
    for b0 in range(0, B, 64):
        out[b0:b0 + 64] = base[:min(64, B - b0)]
    return out, ptr


def wall(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def rate_rows(h, rate, B, n_enrol, steps, warmup, sample, seed, bank_host):
    dev = torch.device("cuda:0")
    L, M = rr.ratio(rate)
    U8 = -(-rate * L // M)
    pcm, p_pcm = captures_at(rate, B, seed)
    y8, p_y8 = pinned((B, U8))
    s = torch.cuda.current_stream()
    d_in = torch.empty((n_enrol, rate), dtype=torch.int16, device=dev)
    d_out = torch.empty((n_enrol, U8), dtype=torch.int16, device=dev)

    def dev_resample(n):
        d_in[:n].copy_(torch.from_numpy(pcm[:n].view(np.int16)), non_blocking=True)
        sr_b200.resample_adc12_dev(d_in.data_ptr(), rate, n, None, rate, d_out.data_ptr(), U8, None, s.cuda_stream)
        torch.from_numpy(y8[:n].view(np.int16)).copy_(d_out[:n], non_blocking=True)
        s.synchronize()
    for b0 in range(0, B, n_enrol):                  # the 8 kHz audio once, by K15 on the device
        n = min(n_enrol, B - b0)
        d_in[:n].copy_(torch.from_numpy(pcm[b0:b0 + n].view(np.int16)))
        sr_b200.resample_adc12_dev(d_in.data_ptr(), rate, n, None, rate, d_out.data_ptr(), U8, None, s.cuda_stream)
        s.synchronize()
        y8[b0:b0 + n] = d_out[:n].cpu().numpy().view(np.uint16)

    def with_mode(mode, fn):
        def run():
            h.set_transport(mode)
            return fn(), h.transport_stats()
        return run
    ep = pcm[:n_enrol]
    calls = {
        "recognise/plain": with_mode(0, lambda: h.recognise(pcm, N_LEN, WANT, rate=rate)),
        "recognise/packed": with_mode(1, lambda: h.recognise(pcm, N_LEN, WANT, rate=rate)),
        "recognise/8k_fed": with_mode(0, lambda: h.recognise(y8, N_LEN, WANT)),
        "enrol/at_rate": lambda: (h.enrol(ep, N_LEN, rate=rate), None),
        "enrol/dev_path": lambda: (dev_resample(n_enrol), h.enrol(y8[:n_enrol], N_LEN))[1:] + (None,),
    }
    for fn in calls.values():
        for _ in range(warmup):
            fn()
    ms = {k: [] for k in calls}
    outs, stats = {}, {}
    for _ in range(steps):                            # alternate the paths, one call each per round
        for k, fn in calls.items():
            t, (outs[k], stats[k]) = wall(fn)
            ms[k].append(t)
    res = {}
    for k, v in ms.items():
        m = float(np.median(v))
        n = n_enrol if k.startswith("enrol") else B
        h2d = stats[k][2] if stats[k] else n * (U8 if k.endswith("dev_path") else rate) * 2
        res[k] = dict(ms=m, ms_all=[round(x, 2) for x in v], captures_per_s=n / (m / 1e3), h2d_GBps=h2d / (m / 1e3) / 1e9,
                      h2d_bytes=h2d)
        if stats[k]:
            res[k]["packed_chunks"], res[k]["plain_chunks"] = stats[k][0], stats[k][1]
    for k in ("recognise/plain", "recognise/packed", "enrol/at_rate"):
        w, recs, _ = timed(h, lambda: calls[k]()[0], steps, 8192)
        ker = per_call(recs, steps)
        res[k].update(resample_ms=ker.get(15, 0.0), resample_share=ker.get(15, 0.0) / w,
                      resample_launches=sum(1 for tag, _ in recs if tag == 15) // steps)
    h.set_transport(-1)
    # equal outputs across the paths, and sampled captures against the CPU composition
    ref = outs["recognise/8k_fed"]
    ok = all(outs[p][f].tobytes() == ref[f].tobytes() for p in ("recognise/plain", "recognise/packed") for f in ref)
    ok &= all(a.tobytes() == b.tobytes() for a, b in zip(outs["enrol/at_rate"], outs["enrol/dev_path"]))
    rng = np.random.default_rng(seed)
    rows = sorted({0, B - 1, *rng.integers(0, B, max(0, sample - 2)).tolist()})
    y = rr.resample_batch(pcm[rows], rate, np.full(len(rows), rate, np.uint32), U8)
    want = ob.port().recognise_batch(y, N_LEN, bank_host, 20, 4096)
    got = outs["recognise/plain"]
    for i, b in enumerate(rows):
        ok &= all(int(np.asarray(got[f][b]).reshape(-1)[0]) == int(np.asarray(want[f][i]).reshape(-1)[0])
                  for f in ("best_idx", "best_dis", "cmd", "status"))
        ok &= got["seg_off"][b].tobytes() == want["seg_off"][i].tobytes()
    for ptr in (p_pcm, p_y8):
        sr_b200.host_free(ptr)
    return res, dict(ok_status=int((got["status"] == 0).sum()), oracle_rows=len(rows)), bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--captures", type=int, default=16384)
    ap.add_argument("--enrol", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    cuda_device("bench_capture_rate")
    h = sr_b200.Handle(0)
    s = torch.cuda.current_stream()
    bank = device_bank(h, s, 20)
    bank_host = bank.cpu().numpy()
    res = dict(card=card(), workload="%d captures x 1 s in pinned host memory, configs[1] bank (20 templates), n_len %d; "
               "enrolment on the first %d" % (a.captures, N_LEN, a.enrol), rows={})
    ok = True
    for rate, seed in ((16000, 0x2D00), (44100, 0x2D01), (48000, 0x2D02)):
        rows, info, good = rate_rows(h, rate, a.captures, min(a.enrol, a.captures), a.steps, a.warmup, a.sample, seed,
                                     bank_host)
        ok &= good
        res["rows"][str(rate)] = dict(paths=rows, oracle_ok=good, **info)
        for k, v in rows.items():
            print("%5d Hz %-17s %8.1f ms  %9.0f captures/s  %6.2f GB/s H2D%s%s" % (
                rate, k, v["ms"], v["captures_per_s"], v["h2d_GBps"],
                "  (%d packed, %d plain)" % (v["packed_chunks"], v["plain_chunks"]) if "packed_chunks" in v else "",
                "  resample %.2f ms (%.1f %%, %d launches)" % (v["resample_ms"], 100 * v["resample_share"],
                                                               v["resample_launches"]) if "resample_ms" in v else ""))
    h.close()
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}))
    report("bench_capture_rate", res, ok, a.json)


if __name__ == "__main__":
    main()
