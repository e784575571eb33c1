"""Throughput of sr_resample_adc12_dev (include/sr_synth.h): 256 recordings of 60 s of random 12-bit codes at 16, 44.1
and 48 kHz, device-resident, resampled to 8 kHz.

Per rate: ms per call from CUDA events around `--steps` calls (after `--warmup`), audio-seconds resampled per second,
the integer multiply-adds per second (out_len * N / L per recording, the taps one output meets on average), and the
achieved bytes/s (2 B read per input sample, 2 B written per output) against the H100 SXM's 3.35 TB/s of HBM3. The
outputs of sampled recordings are checked against tests/resample_ref.py on sampled windows. The card's name, power
limit and SM clock limit are read in the same run.

    python tools/bench_resample.py [--recordings 256] [--seconds 60] [--steps 10] [--warmup 2] [--json FILE]
"""
import argparse
import json

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import HBM_PEAK, card, cuda_device, event_steps, report
import resample_ref as rr
import sr_b200


def row(rate, B, secs, steps, warmup, sample, seed):
    dev = torch.device("cuda:0")
    U_in = rate * secs
    L, M = rr.ratio(rate)
    U_out = rr.out_len(U_in, rate)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    x = torch.randint(0, 4096, (B, U_in), dtype=torch.int16, device=dev, generator=g)
    out = torch.zeros((B, U_out), dtype=torch.int16, device=dev)
    olens = torch.zeros(B, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream()

    def call():
        sr_b200.resample_adc12_dev(x.data_ptr(), U_in, B, None, rate, out.data_ptr(), U_out, olens.data_ptr(), s.cuda_stream)
    ms, _ = event_steps(None, s, call, steps, warmup)
    # sampled check: first, last and two random recordings; their first and last 4096 outputs and 4 random windows
    rng = np.random.default_rng(seed)
    rows = sorted({0, B - 1, *rng.integers(0, B, 2).tolist()})
    ok = bool((olens.cpu().numpy() == U_out).all())
    for b in rows:
        xb = x[b].cpu().numpy().view(np.uint16)
        starts = [0, U_out - 4096, *rng.integers(0, U_out - 4096, 4).tolist()]
        idx = np.unique(np.concatenate([np.arange(a, a + 4096) for a in starts]))
        got = out[b].cpu().numpy().view(np.uint16)[idx]
        ok = ok and np.array_equal(got, rr.resample(xb, rate, idx))
    nbytes = 2 * B * (U_in + U_out)
    macs = B * U_out * len(rr.taps(rate)) / L
    del x, out
    torch.cuda.empty_cache()
    return dict(rate=rate, B=B, seconds=secs, ms_per_call=ms, audio_s_per_s=B * secs / (ms / 1e3),
                Gmac_per_s=macs / (ms / 1e3) / 1e9, GBps=nbytes / (ms / 1e3) / 1e9,
                share_of_hbm=nbytes / (ms / 1e3) / HBM_PEAK, oracle_ok=ok, oracle_rows=len(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=256)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--rates", default="16000,44100,48000")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    cuda_device("bench_resample")
    res = dict(card=card(), rows={})
    for rate in (int(r) for r in a.rates.split(",")):
        res["rows"]["%dHz" % rate] = row(rate, a.recordings, a.seconds, a.steps, a.warmup, a.sample, 0x5E5A + rate)
    for k, v in res["rows"].items():
        print(k, json.dumps(v))
    report("bench_resample", res, all(v["oracle_ok"] for v in res["rows"].values()), a.json)


if __name__ == "__main__":
    main()
