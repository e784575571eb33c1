"""Throughput of the connected-word calls (K6): sr_connected_batch and sr_recognise_connected_batch.

  1. sr_connected_batch on 65 536 synthetic feature sequences at N in {119, 300, 818} frames against banks of 20 and 80
     signed slots (synthetic templates of 50..100 frames): the decoder kernel's time (tag 9), sequences/s and cells/s,
     cells = N * sum of the members' frame counts; the host call's wall time too (it moves B * N * 24 bytes of features).
  2. sr_recognise_connected_batch on synthetic 3-word captures at U = 16 000 against an enrolled 80-slot bank: wall time
     per call and the kernel time by tag (0 noise_atap + VAD, 1 get_mfcc pieces, 9 the decoder).

Every row checks a sample against the oracles (tests/oracle_ext/connected.c, the composed oracle stages): the first and last
sequence (capture) of every launch -- decoder launches of 2^20 sequences, get_mfcc piece launches of 8 192 pieces -- plus
random ones, --sample in all. The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_connected.py [--steps 2] [--warmup 1] [--json FILE]
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
from test_connected_launches import _pieces, launch_sample, piece_plan, seq_launches  # noqa: E402

NPROC = os.cpu_count() or 1
PENALTY = 4000


def edges(ranges):
    """the first and last index of every range [lo, hi)"""
    return {i for lo, hi in ranges for i in (lo, hi - 1)}


def e2e_edges(frm_num, seq_ranges=None):
    """the captures holding the first and last get_mfcc piece of every piece launch and, given the decoder's launch ranges
    over the captures' segments with frames (default: one sequence per segment, K6), of every decoder launch"""
    B = len(frm_num)
    e = piece_plan(_pieces(frm_num).sum(1))[1]
    if seq_ranges is None:
        owner = np.repeat(np.arange(B), (frm_num > 0).sum(1))
        e |= {int(owner[i]) for i in edges(seq_launches([0, len(owner)]))}
    else:
        e |= edges(seq_ranges)
    return e


def timed(h, fn, reps):
    """(wall ms per call, {tag: kernel ms per call}, last result) of fn() repeated reps times"""
    h.timing_enable(4096 * reps)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    ker = {}
    for t, ms in h.timing_collect():
        ker[t] = ker.get(t, 0.0) + ms / reps
    h.timing_enable(0)
    return wall, ker, out


def synth_bank(T, seed):
    ftr = sr_b200.synth_ftr_host(T, seed, 50, 100).view(ob.FTR_DTYPE).reshape(T)
    return sr_b200.make_bank(ftr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--e2e-batch", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=32)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_connected: no CUDA device (there is nothing to measure without one)")
    B, n = args.batch, args.sample
    h = sr_b200.Handle(0)
    co = ox.connected()
    results = {"decoder": [], "end_to_end": []}

    # 1. the decoder: sequences of synthetic feature rows (2 000 structs of 50..100 frames, rows drawn at random)
    pool = sr_b200.synth_ftr_host(2000, 0xB0C0000, 50, 100).view(ob.FTR_DTYPE).reshape(2000)
    rows = np.concatenate([pool["mfcc_dat"][k][:int(pool["frm_num"][k]) * 12].reshape(-1, 12) for k in range(2000)])
    rng = np.random.default_rng(0xB0C)
    srng = np.random.default_rng(0xB0C5)                  # the oracle samples' random part
    for N in (119, 300, 818):
        start = rng.integers(0, len(rows) - N, B)
        feat = np.empty((B, N, 12), np.int16)
        for b0 in range(0, B, 4096):
            idx = start[b0:b0 + 4096, None] + np.arange(N)[None, :]
            feat[b0:b0 + 4096] = rows[idx]
        frm = np.full(B, N, np.uint32)
        for T in (20, 80):
            bank = synth_bank(T, 0xB0C1000 + T)
            h.set_bank(bank, T, 4096)
            for _ in range(args.warmup):
                h.connected(feat, frm, PENALTY, 16)
            wall, ker, (words, nw, tot) = timed(h, lambda: h.connected(feat, frm, PENALTY, 16), args.steps)
            idx = launch_sample(edges(seq_launches([0, B])), B, n, srng)
            ww, wn, wt = co.connected(feat[idx], frm[idx], bank, T, 4096, PENALTY, 16, nthreads=NPROC)
            ok = bool(np.array_equal(nw[idx], wn) and np.array_equal(tot[idx], wt) and np.array_equal(words[idx], ww))
            cells = float(N) * float(bank[:, 2:4].copy().view(np.uint16)[:, 0].astype(np.int64).sum()) * B
            kms = ker[9]
            results["decoder"].append({"N": N, "slots": T, "sequences": B, "kernel_ms": kms, "wall_ms": wall,
                                       "sequences_per_s": B / (kms * 1e-3), "cells_per_s": cells / (kms * 1e-3),
                                       "mean_words": float(nw.mean()), "sample_equals_oracle": ok})
        del feat

    # 2. end to end: synthetic 3-word captures, an 80-slot bank of enrolled one-word captures (20 commands x 4)
    U, E = 16000, args.e2e_batch
    bank, st = h.enrol(sr_b200.synth_pcm_host(80, 8000, 0xB0C2000), 2400)
    h.set_bank(bank, 80, 4096)
    pcm = sr_b200.synth_pcm_host(E, U, 0xB0C3000, 3)
    for _ in range(args.warmup):
        h.recognise_connected(pcm, PENALTY, 8)
    wall, ker, out = timed(h, lambda: h.recognise_connected(pcm, PENALTY, 8), args.steps)
    idx = launch_sample(e2e_edges(out["frm_num"]), E, n, srng)
    want = ox.recognise_connected(ob.best_oracle(), co, pcm[idx], 2400, bank, 80, 4096, PENALTY, 8)
    ok = all(np.array_equal(out[k][idx], want[k]) for k in ("seg_off", "frm_num", "n_words", "total", "status", "words"))
    results["end_to_end"].append({"U": U, "captures": E, "wall_ms": wall, "captures_per_s": E / (wall * 1e-3),
                                  "kernel_ms": {str(k): v for k, v in sorted(ker.items())},
                                  "mean_words": float(out["n_words"].mean()), "sample_equals_oracle": bool(ok)})

    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "penalty": PENALTY, "steps": args.steps,
            "sample": n, "results": results}
    c = info["card"]
    print("card: %s, power limit %s, max SM clock %s" % (c.get("name"), c.get("power.limit"), c.get("clocks.max.sm")))
    for x in results["decoder"]:
        print("decoder N=%-4d slots=%-3d kernel %9.2f ms  wall %9.1f ms  %8.3f Mseq/s  %7.2f Gcells/s  %.2f words  oracle %s" % (
            x["N"], x["slots"], x["kernel_ms"], x["wall_ms"], x["sequences_per_s"] / 1e6, x["cells_per_s"] / 1e9,
            x["mean_words"], x["sample_equals_oracle"]))
    for x in results["end_to_end"]:
        print("end to end U=%d B=%d  wall %9.1f ms  %9.0f captures/s  kernels %s  %.2f words  oracle %s" % (
            x["U"], x["captures"], x["wall_ms"], x["captures_per_s"], x["kernel_ms"], x["mean_words"], x["sample_equals_oracle"]))
    print(json.dumps(info))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    h.close()
    if not all(x["sample_equals_oracle"] for v in results.values() for x in v):
        raise SystemExit("bench_connected: a sample differs from the oracle")


if __name__ == "__main__":
    main()
