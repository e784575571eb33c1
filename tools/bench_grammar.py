"""Throughput of the grammar decoder (K6g): sr_connected_grammar_batch and sr_recognise_connected_grammar_batch.

  1. overhead: the loop grammar against sr_connected_batch on 65 536 sequences of 119 frames against 20 signed slots,
     the two calls alternated in one run (tag 10 against tag 9);
  2. 4-digit chain: the PIN grammar against an averaged 10-digit bank (40 copies), 16 384 sequences of 300 frames;
  3. 11-digit chain: 12 states, 110 copies (11 digit states of 10 averaged digits), sequences of 818 frames;
  4. end to end: 16 384 two-second captures under the PIN grammar.
Kernel time (tags 9 and 10), sequences/s and cells/s, cells = N * sum of the copies' frame counts. Every row checks a
sample against the oracle (tests/oracle_ext/long_grammar.c, the composed oracle stages): the first and last sequence (capture) of
every launch -- decoder launches cut at 2^28 bytes of records and at 2^20 sequences, get_mfcc piece launches of 8 192
pieces -- plus random ones, --sample in all. The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_grammar.py [--steps 2] [--warmup 1] [--json FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "stm32-speech-recognition_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import oracle_bind as ob  # noqa: E402
import oracle_ext as ox  # noqa: E402
import sr_b200  # noqa: E402
from bench_connected import e2e_edges, edges, synth_bank, timed  # noqa: E402
from bench_match import card  # noqa: E402
from test_connected_launches import launch_sample, record_cuts, seq_launches  # noqa: E402

NPROC = os.cpu_count() or 1
PENALTY = 4000
PIN = (5, 1 << 4, [(k, k + 1, 0x3FF) for k in range(4)])
PHONE = (12, 1 << 11, [(k, k + 1, 0x3FF) for k in range(11)])


def copy_frames(bank, grammar):
    """sum of the copies' frame counts (the cells per input frame)"""
    S, _, arcs = grammar
    hdr = bank[:, :4].copy().view(np.uint16)
    tot = 0
    for s in range(S):
        for t in range(len(bank)):
            if hdr[t, 0] == sr_b200.SAVE_MASK and 1 <= hdr[t, 1] <= 119 and any(b == s and (m >> (t // 4)) & 1 for _, b, m in arcs):
                tot += int(hdr[t, 1])
    return tot


def features(B, N, seed):
    pool = sr_b200.synth_ftr_host(2000, seed, 50, 100).view(ob.FTR_DTYPE).reshape(2000)
    rows = np.concatenate([pool["mfcc_dat"][k][:int(pool["frm_num"][k]) * 12].reshape(-1, 12) for k in range(2000)])
    rng = np.random.default_rng(seed)
    start = rng.integers(0, len(rows) - N, B)
    feat = np.empty((B, N, 12), np.int16)
    for b0 in range(0, B, 4096):
        feat[b0:b0 + 4096] = rows[start[b0:b0 + 4096, None] + np.arange(N)[None, :]]
    return feat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--chain-batch", type=int, default=16384)
    ap.add_argument("--phone-batch", type=int, default=4096)
    ap.add_argument("--e2e-batch", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=32)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_grammar: no CUDA device (there is nothing to measure without one)")
    n = args.sample
    h = sr_b200.Handle(0)
    go = ox.grammar()
    rows = []
    srng = np.random.default_rng(0xB6A5)                  # the oracle samples' random part

    def row(name, B, N, bank, T, grammar, kms, words, nw, tot, feat, frm):
        idx = launch_sample(edges(seq_launches(record_cuts(frm, grammar[0]))), B, n, srng)
        ww, wn, wt = go.decode(feat[idx], frm[idx], bank, T, 4096, grammar, PENALTY, 16, nthreads=NPROC)
        ok = bool(np.array_equal(nw[idx], wn) and np.array_equal(tot[idx], wt) and np.array_equal(words[idx], ww))
        cells = float(N) * copy_frames(bank, grammar) * B
        rows.append({"row": name, "sequences": B, "N": N, "states": grammar[0], "kernel_ms": kms,
                     "sequences_per_s": B / (kms * 1e-3), "cells_per_s": cells / (kms * 1e-3),
                     "mean_words": float(nw.mean()), "sample_equals_oracle": ok})

    # 1. overhead of the loop grammar over K6, alternated
    B = args.batch
    feat = features(B, 119, 0xB6A0000)
    frm = np.full(B, 119, np.uint32)
    bank = synth_bank(20, 0xB6A1000)
    h.set_bank(bank, 20, 4096)
    loop = sr_b200.loop_grammar()
    for _ in range(args.warmup):
        h.connected(feat, frm, PENALTY, 16)
        h.connected_grammar(feat, frm, loop, PENALTY, 16)
    k6, k6g = [], []
    for _ in range(args.steps):
        _, ker, out_k6 = timed(h, lambda: h.connected(feat, frm, PENALTY, 16), 1)
        k6.append(ker[9])
        _, ker, out = timed(h, lambda: h.connected_grammar(feat, frm, loop, PENALTY, 16), 1)
        k6g.append(ker[10])
    same = all(np.array_equal(a, b) for a, b in zip(out_k6, out))
    row("loop grammar", B, 119, bank, 20, loop, float(np.median(k6g)), *out, feat, frm)
    rows[-1]["k6_kernel_ms"] = float(np.median(k6))
    rows[-1]["overhead"] = float(np.median(k6g)) / float(np.median(k6)) - 1
    rows[-1]["equals_connected_batch"] = bool(same)
    rows[-1]["sample_equals_oracle"] &= same
    del feat

    # averaged digit bank: 10 digits x 4 enrolled captures, averaged into slot 4 * digit
    enr, _ = h.enrol(sr_b200.synth_pcm_host(40, 8000, 0xB6A2000), 2400)
    avg = h.average_bank(enr, 4096, 4, 118, 2)[0]
    h.set_bank(avg, 40, 4096)
    # 2. 4-digit chain, 40 copies
    for name, g, B, N in (("4-digit chain", PIN, args.chain_batch, 300), ("11-digit chain", PHONE, args.phone_batch, 818)):
        feat = features(B, N, 0xB6A3000 + N)
        frm = np.full(B, N, np.uint32)
        for _ in range(args.warmup):
            h.connected_grammar(feat, frm, g, PENALTY, 16)
        _, ker, out = timed(h, lambda: h.connected_grammar(feat, frm, g, PENALTY, 16), args.steps)
        row(name, B, N, avg, 40, g, ker[10], *out, feat, frm)
        del feat

    # 4. end to end under the PIN grammar
    U, E = 16000, args.e2e_batch
    pcm = sr_b200.synth_pcm_host(E, U, 0xB6A4000, 3)
    for _ in range(args.warmup):
        h.recognise_connected_grammar(pcm, PIN, PENALTY, 8)
    wall, ker, out = timed(h, lambda: h.recognise_connected_grammar(pcm, PIN, PENALTY, 8), args.steps)
    idx = launch_sample(e2e_edges(out["frm_num"], seq_launches(record_cuts(out["frm_num"].sum(1), PIN[0]))), E, n, srng)
    want = ox.recognise_connected_grammar(ob.best_oracle(), go, pcm[idx], 2400, avg, 40, 4096, PIN, PENALTY, 8, nthreads=NPROC)
    ok = all(np.array_equal(out[k][idx], want[k]) for k in ("seg_off", "frm_num", "n_words", "total", "status", "words"))
    e2e = {"U": U, "captures": E, "wall_ms": wall, "captures_per_s": E / (wall * 1e-3),
           "kernel_ms": {str(k): v for k, v in sorted(ker.items())}, "mean_words": float(out["n_words"].mean()),
           "sample_equals_oracle": bool(ok)}

    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "penalty": PENALTY, "steps": args.steps,
            "sample": n, "decoder": rows, "end_to_end": e2e}
    c = info["card"]
    print("card: %s, power limit %s, max SM clock %s" % (c.get("name"), c.get("power.limit"), c.get("clocks.max.sm")))
    for x in rows:
        extra = "  K6 %.2f ms, overhead %+.1f %%" % (x["k6_kernel_ms"], 100 * x["overhead"]) if "overhead" in x else ""
        print("%-15s B=%-6d N=%-4d S=%-2d kernel %9.2f ms  %8.3f Mseq/s  %7.2f Gcells/s  %.2f words  oracle %s%s" % (
            x["row"], x["sequences"], x["N"], x["states"], x["kernel_ms"], x["sequences_per_s"] / 1e6, x["cells_per_s"] / 1e9,
            x["mean_words"], x["sample_equals_oracle"], extra))
    print("end to end U=%d B=%d  wall %9.1f ms  %9.0f captures/s  kernels %s  %.2f words  oracle %s" % (
        e2e["U"], e2e["captures"], e2e["wall_ms"], e2e["captures_per_s"], e2e["kernel_ms"], e2e["mean_words"],
        e2e["sample_equals_oracle"]))
    print(json.dumps(info))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    h.close()
    if not (all(x["sample_equals_oracle"] for x in rows) and e2e["sample_equals_oracle"]):
        raise SystemExit("bench_grammar: a sample differs from the oracle")


if __name__ == "__main__":
    main()
