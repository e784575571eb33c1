"""Throughput of the host-buffer long-form calls at a rate (sr_recognise_long_batch_at_rate and
sr_recognise_long_grammar_batch_at_rate, include/sr_synth.h): 256 recordings of 60 s at 48 kHz and at 44.1 kHz in pinned
host memory, against bench.py's configs[1] bank (20 templates synthesised on the device).

Per rate, alternating in one run, `--steps` calls of each (after `--warmup`):
  at_rate      the call at the rate: the input crosses PCIe once and K15 runs per staged group (tag 15);
  8k_fed       the 8 kHz host call on the same audio resampled beforehand: the same kernels without K15, a sixth (48 kHz)
               or 18 % (44.1 kHz) of the bytes to copy;
  dev_path     the grammar call only: the path it had before, K15 on a device copy of the whole batch, the 8 kHz audio
               back to pinned host memory, then the 8 kHz host call (three PCIe passes).
Reported: wall ms per call (host clock around calls that end in a synchronisation), audio-seconds per second, the input
bytes the call copies host to device per second of the call, and tag 15's share of the at-rate call (its kernel time
over the call's wall time) and kernel ms per call by timing tag (13 the grammar decoder), both from separate timed
windows. Sampled recordings are checked against the CPU composition:
tests/resample_ref.py, then the long-form oracles. The card's name, power limit and SM clock limit are read in the same
run.

    python tools/bench_long_rate.py [--recordings 256] [--seconds 60] [--steps 3] [--warmup 1] [--json FILE]
"""
import argparse
import json
import time

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import card, cuda_device, device_bank, per_call, report, timed
import oracle_bind as ob
import oracle_ext as ox
import resample_ref as rr
import sr_b200

MAX_SEGS, MAX_WORDS, N_LEN, PENALTY = 64, 256, 2400, 1000
LOOP = sr_b200.loop_grammar()


def pinned(shape):
    mem, ptr = sr_b200.host_alloc_dev(0, int(np.prod(shape)) * 2)
    return mem.view(np.uint16).reshape(shape), ptr


def audio_at(rate, B, secs, seed):
    """B synthetic recordings at 8 kHz (ox.synth_long) taken to `rate` by linear interpolation, in pinned memory"""
    U8, U_in = 8000 * secs, rate * secs
    x8 = ox.synth_long(B, U8, seed)
    out, ptr = pinned((B, U_in))
    t = np.arange(U_in) * (8000.0 / rate)
    for b in range(B):
        out[b] = np.rint(np.interp(t, np.arange(U8), x8[b])).astype(np.uint16)
    return out, ptr


def wall(fn, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        out = fn()
    return (time.perf_counter() - t0) * 1e3 / steps, out


def rate_rows(h, rate, B, secs, steps, warmup, sample, seed, bank_host):
    dev = torch.device("cuda:0")
    U_in = rate * secs
    L, M = rr.ratio(rate)
    U8 = -(-U_in * L // M)
    pcm, p_pcm = audio_at(rate, B, secs, seed)
    # the 8 kHz audio once, by K15 on the device, into pinned memory
    y8, p_y8 = pinned((B, U8))
    d_in = torch.empty((B, U_in), dtype=torch.int16, device=dev)
    d_out = torch.empty((B, U8), dtype=torch.int16, device=dev)
    s = torch.cuda.current_stream()

    def dev_resample():
        d_in.copy_(torch.from_numpy(pcm.view(np.int16)), non_blocking=True)
        sr_b200.resample_adc12_dev(d_in.data_ptr(), U_in, B, None, rate, d_out.data_ptr(), U8, None, s.cuda_stream)
        torch.from_numpy(y8.view(np.int16)).copy_(d_out, non_blocking=True)
        s.synchronize()
    dev_resample()
    calls = {
        "long/at_rate": lambda: h.recognise_long_batch(pcm, MAX_SEGS, N_LEN, rate=rate),
        "long/8k_fed": lambda: h.recognise_long_batch(y8, MAX_SEGS, N_LEN),
        "grammar/at_rate": lambda: h.recognise_long_grammar(pcm, LOOP, PENALTY, MAX_SEGS, MAX_WORDS, N_LEN, rate=rate),
        "grammar/8k_fed": lambda: h.recognise_long_grammar(y8, LOOP, PENALTY, MAX_SEGS, MAX_WORDS, N_LEN),
        "grammar/dev_path": lambda: (dev_resample(), h.recognise_long_grammar(y8, LOOP, PENALTY, MAX_SEGS, MAX_WORDS, N_LEN))[1],
    }
    for fn in calls.values():
        for _ in range(warmup):
            fn()
    ms = {k: [] for k in calls}
    outs = {}
    for _ in range(steps):                        # alternate the paths, one call each per round
        for k, fn in calls.items():
            t, outs[k] = wall(fn, 1)
            ms[k].append(t)
    res = {}
    audio_s = B * secs
    for k, v in ms.items():
        m = float(np.median(v))
        h2d = B * (U8 if "8k_fed" in k else U_in) * 2           # the input each call copies host to device
        pcie = h2d + (4 * B * U8 if k.endswith("dev_path") else 0)     # dev_path: + the 8 kHz audio back and in again
        res[k] = dict(ms=m, ms_all=[round(x, 2) for x in v], audio_s_per_s=audio_s / (m / 1e3),
                      h2d_GBps=h2d / (m / 1e3) / 1e9, pcie_bytes=pcie)
    # kernel ms per call by timing tag, and tag 15's share of each at-rate call, in windows of their own
    for k in ("long/at_rate", "long/8k_fed", "grammar/at_rate", "grammar/8k_fed"):
        w, recs, _ = timed(h, calls[k], steps, 4096)
        ker = per_call(recs, steps)
        res[k]["kernel_ms_by_tag"] = {str(t): round(v, 3) for t, v in sorted(ker.items())}
        if k.endswith("at_rate"):
            res[k].update(resample_ms=ker.get(15, 0.0), resample_share=ker.get(15, 0.0) / w,
                          resample_launches=sum(1 for tag, _ in recs if tag == 15) // steps)
    # equal outputs across the paths, and sampled recordings against the CPU composition
    ok = all(outs["long/at_rate"][f].tobytes() == outs["long/8k_fed"][f].tobytes() for f in outs["long/at_rate"])
    ok &= all(outs["grammar/at_rate"][f].tobytes() == outs[p][f].tobytes() for p in ("grammar/8k_fed", "grammar/dev_path")
              for f in outs["grammar/at_rate"])
    rng = np.random.default_rng(seed)
    rows = sorted({0, B - 1, *rng.integers(0, B, max(0, sample - 2)).tolist()})
    lo, port = ox.long_oracle(), ob.port()
    got = outs["long/at_rate"]
    for b in rows:
        y = rr.resample(pcm[b], rate)[None]
        want = ox.recognise_long(lo, port, y, N_LEN, bank_host, 20, 4096, MAX_SEGS)
        m = min(int(want["n_segs"][0]), MAX_SEGS)
        ok &= int(got["n_segs"][b]) == int(want["n_segs"][0]) and got["atap"][b].tobytes() == want["atap"][0].tobytes()
        ok &= got["segs"][b, :m].tobytes() == want["segs"][0, :m].tobytes()
    segs = int(got["n_segs"].sum())
    words = int(outs["grammar/at_rate"]["n_words"].sum())
    for ptr in (p_pcm, p_y8):
        sr_b200.host_free(ptr)
    return res, dict(segments=segs, words=words, oracle_rows=len(rows)), bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=256)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    cuda_device("bench_long_rate")
    h = sr_b200.Handle(0)
    s = torch.cuda.current_stream()
    bank = device_bank(h, s, 20)
    bank_host = bank.cpu().numpy()
    res = dict(card=card(), workload="%d recordings x %d s in pinned host memory, configs[1] bank (20 templates), "
               "max_segs %d, loop grammar, max_words %d" % (a.recordings, a.seconds, MAX_SEGS, MAX_WORDS), rows={})
    ok = True
    for rate, seed in ((48000, 0x1B00), (44100, 0x1B01)):
        rows, info, good = rate_rows(h, rate, a.recordings, a.seconds, a.steps, a.warmup, a.sample, seed, bank_host)
        ok &= good
        res["rows"][str(rate)] = dict(paths=rows, oracle_ok=good, **info)
        for k, v in rows.items():
            print("%5d Hz %-17s %9.1f ms  %9.0f audio-s/s  %6.2f GB/s H2D  decoder %5.1f ms%s" % (
                rate, k, v["ms"], v["audio_s_per_s"], v["h2d_GBps"], v.get("kernel_ms_by_tag", {}).get("13", 0.0),
                "  resample %.1f ms (%.1f %%, %d launches)" % (v["resample_ms"], 100 * v["resample_share"], v["resample_launches"])
                if "resample_ms" in v else ""))
    h.close()
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}))
    report("bench_long_rate", res, ok, a.json)


if __name__ == "__main__":
    main()
