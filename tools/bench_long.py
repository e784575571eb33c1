"""Throughput of the long-form calls (include/sr_long.h).

  1. VAD passes, device PCM (sr_vad_long_batch_dev): one recording of 2^27 samples (4.6 h) and 4 096 recordings of 30 s;
     recording-hours per second of the block pass + segment pass, and the block pass's achieved bytes/s (2 B read per
     sample, 8 B written per 80-sample block) against the H100 SXM's 3.35 TB/s of HBM3;
  2. end to end (sr_recognise_long_batch, host buffers): 4 096 recordings of 30 s against a 12-slot bank, segments/s.
Kernel times come from the timing tags (11 block pass: its noise_atap launch, then the block summaries; 12 segment pass),
wall times from a host clock around calls that end in a synchronisation. Every row checks the oracle: the VAD of every
recording (tests/oracle_ext/long.c), and the per-segment records of sampled recordings (tests/oracle_ext.py). The card's
name, power limit and SM clock limit are read in the same run.

    python tools/bench_long.py [--steps 3] [--warmup 1] [--json FILE]
"""
import argparse
import json
import time

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import HBM_PEAK, card, cuda_device, report, timed
import oracle_bind as ob
import oracle_ext as ox
import sr_b200


def vad_row(h, B, U, seed, steps, warmup, max_segs):
    """one VAD configuration on device-resident PCM: timings and the oracle check of every recording"""
    dev = torch.device("cuda:0")
    pcm = ox.synth_long(B, U, seed)
    d_pcm = torch.from_numpy(pcm.view(np.int16)).to(dev)
    d_atap = torch.zeros(B * 12, dtype=torch.uint8, device=dev)
    d_n = torch.zeros(B, dtype=torch.int32, device=dev)
    d_seg = torch.zeros(B * max_segs * 2, dtype=torch.int32, device=dev)

    def call():
        h.vad_long_batch_dev(d_pcm.data_ptr(), U, B, None, 2400, max_segs, d_atap.data_ptr(), d_n.data_ptr(), d_seg.data_ptr())
    for _ in range(warmup):
        call()
    wall, rec, _ = timed(h, call, steps, 8 * steps)
    assert [t for t, _ in rec] == [11, 11, 12] * steps, rec
    atap_ms = sum(ms for k, (_, ms) in enumerate(rec) if k % 3 == 0) / steps
    block_ms = sum(ms for k, (_, ms) in enumerate(rec) if k % 3 == 1) / steps
    seg_ms = sum(ms for k, (_, ms) in enumerate(rec) if k % 3 == 2) / steps
    # oracle: every recording
    atap = d_atap.cpu().numpy().view(ob.ATAP_DTYPE)
    n, seg = ox.long_oracle().vad_long(pcm, atap, max_segs)
    got_n = d_n.cpu().numpy().view(np.uint32)
    got_seg = d_seg.cpu().numpy().view(np.uint32).reshape(B, max_segs, 2)
    want_atap = ox.atap_long(ob.port(), pcm[: min(B, 64)], 2400)
    ok = (got_n == n).all() and (got_seg == seg).all() and atap[: min(B, 64)].tobytes() == want_atap.tobytes()
    hours = B * U / 8000 / 3600
    nblk = B * (U // 80 + 1)
    block_bytes = B * U * 2 + nblk * 8
    return dict(B=B, U=U, segments=int(got_n.sum()), wall_ms=wall, atap_ms=atap_ms, block_ms=block_ms, segment_ms=seg_ms,
                vad_hours_per_s=hours / ((atap_ms + block_ms + seg_ms) / 1e3),
                block_GBps=block_bytes / (block_ms / 1e3) / 1e9, block_share_of_hbm=block_bytes / (block_ms / 1e3) / HBM_PEAK,
                oracle_ok=bool(ok), oracle_rows=B)


def e2e_row(h, B, U, seed, steps, warmup, max_segs, sample):
    pcm = ox.synth_long(B, U, seed)
    tpl = sr_b200.synth_pcm_host(12, 8000, 0x7E3A0000)
    e = ob.port().recognise_batch(tpl, 2400, None, 0, 4096)
    bank = sr_b200.make_bank(e["ftr"])
    h.set_bank(bank, 12, 4096)
    for _ in range(warmup):
        got = h.recognise_long_batch(pcm, max_segs, 2400)
    t0 = time.perf_counter()
    for _ in range(steps):
        got = h.recognise_long_batch(pcm, max_segs, 2400)
    wall = (time.perf_counter() - t0) / steps
    nseg = int(np.minimum(got["n_segs"], max_segs).sum())
    rng = np.random.default_rng(seed)
    rows = sorted({0, B - 1, *rng.integers(0, B, sample - 2).tolist()})
    lo, port = ox.long_oracle(), ob.port()
    want = ox.recognise_long(lo, port, pcm, 2400, bank, 12, 4096, max_segs, rows=rows)
    n, _ = lo.vad_long(pcm, got["atap"], max_segs)
    ok = (got["n_segs"] == n).all() and all(
        got["segs"][b].tobytes() == want["segs"][b].tobytes() and got["atap"][b].tobytes() == want["atap"][b].tobytes() for b in rows)
    return dict(B=B, U=U, segments=nseg, wall_ms=wall * 1e3, segments_per_s=nseg / wall,
                recording_hours_per_s=B * U / 8000 / 3600 / wall, oracle_ok=bool(ok), oracle_rows=len(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=16)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    cuda_device("bench_long")
    h = sr_b200.Handle(0)
    res = dict(card=card(), rows={})
    res["rows"]["vad_1x2^27"] = vad_row(h, 1, 1 << 27, 0xB10, a.steps, a.warmup, 32768)
    res["rows"]["vad_4096x30s"] = vad_row(h, 4096, 240000, 0xB20, a.steps, a.warmup, 64)
    res["rows"]["e2e_4096x30s"] = e2e_row(h, 4096, 240000, 0xB20, a.steps, a.warmup, 64, a.sample)
    h.close()
    for k, v in res["rows"].items():
        print(k, json.dumps(v))
    report("bench_long", res, all(v["oracle_ok"] for v in res["rows"].values()), a.json)


if __name__ == "__main__":
    main()
