"""Recognition time without a decision rule and under the decision rules of sr_set_match -- the runner-up margin rule
SR_DTW_REJECT(q) and the KNN rule SR_DTW_KNN(k), alone or together -- under the greedy walk and the banded DP at r = 10
and r = 118, on BASELINE configs[1]'s shape (65 536 utterances x 1 s, synthetic PCM generated on the device) against
banks of 20 and 80 templates. The default rows cover both rules' cost tables in DESIGN.md.

Per (bank, matcher, k, q): W warm-up steps, then K steps of sr_recognise_batch_dev between CUDA events (ms/step), and the
library's own event pairs (sr_timing_*) for best-init (tag 3), the template scan (4 greedy / 6 banded) and the finisher
(tag 5), which under a rule reads the per-command (margin rule) or per-slot (KNN) keys. Every setting of a bank is warmed
up before any is timed, and the settings alternate, several rounds. A sample of every row's outputs -- the first
utterances of the launch and its last ones -- is checked against the oracle: its front end (recognise_pinned), its
template scan under the same matcher (match_scores), then the rule in numpy (refs.decide). The card's name, power limit
and SM clock limit are read in the same run.

    python tools/bench_rule.py [--templates 20,80] [--rules 0:0,0:100,2:0,3:0,4:0] [--steps 20] [--warmup 3]
                               [--rounds 2] [--json FILE]
"""
import argparse

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import N_LEN, SEED, U, card, cuda_device, device_bank, event_steps, report, sample_rows
import oracle_bind as ob
import oracle_ext as ox
import sr_b200
from refs import decide

MATCHERS = ((0, 0), (sr_b200.DTW_BAND, 10), (sr_b200.DTW_BAND, 118))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--templates", default="20,80")
    ap.add_argument("--rules", default="0:0,0:100,2:0,3:0,4:0", help="k:q of each setting (0:0: no rule)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the settings per bank")
    ap.add_argument("--sample", type=int, default=256, help="first utterances checked against the oracle")
    ap.add_argument("--tail", type=int, default=32, help="last utterances checked against the oracle")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    rules = [tuple(int(v) for v in x.split(":")) for x in args.rules.split(",")]

    dev = cuda_device("bench_rule")
    B, n = args.batch, min(args.sample, args.batch)
    stream = torch.cuda.Stream(dev)
    h = sr_b200.Handle(0)
    h.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        pcm = torch.empty((B, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(pcm.data_ptr(), B, U, SEED, 1, stream.cuda_stream)
    rows = sample_rows(B, n, args.tail)
    stream.synchronize()
    sample_pcm = pcm[torch.from_numpy(rows).to(dev)].cpu().numpy().view(np.uint16)
    front = ob.recognise_pinned(ob.best_oracle(), sample_pcm, N_LEN, None, 0, 4096)
    good = front["status"] == 0
    results = []
    for T in [int(x) for x in args.templates.split(",")]:
        bank = device_bank(h, stream, T)
        with torch.cuda.stream(stream):
            outs = {k: torch.zeros(shape, dtype=dt, device=dev) for k, shape, dt in
                    (("seg_off", (B, 6), torch.int32), ("ftr", (B, 2860), torch.uint8), ("score", (B, T), torch.int32),
                     ("best_idx", (B,), torch.int32), ("best_dis", (B,), torch.int32), ("cmd", (B,), torch.int32),
                     ("status", (B,), torch.uint8))}
        ptrs = {k: v.data_ptr() for k, v in outs.items()}
        bank_h = bank.cpu().numpy()
        scores = {}

        def run(flags, r, k, q):
            h.set_match(flags | sr_b200.dtw_knn(k) | sr_b200.dtw_reject(q), r)
            step_ms, recs = event_steps(h, stream, lambda: h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs),
                                        args.steps, args.warmup, 6 * args.steps + 8)
            scan = 6 if flags else 4
            per = {t: [ms for tt, ms in recs if tt == t] for t in (3, scan, 5)}
            assert all(len(v) == args.steps for v in per.values()), (flags, r, k, q, {t: len(v) for t, v in per.items()})
            idx = torch.from_numpy(rows).to(dev)
            got = {key: outs[key][idx].cpu().numpy() for key in ("score", "best_idx", "best_dis", "cmd", "status")}
            got["score"] = got["score"].view(np.uint32)
            if (flags, r) not in scores:
                scores[flags, r] = ox.match_scores(front["ftr"][good], bank_h, T, flags, r)
            sc = scores[flags, r]
            i, d1, cmd, rej = decide(sc, k, q)
            st = front["status"].copy()
            st[np.flatnonzero(good)[rej]] = sr_b200.ST_REJECT
            ok = (np.array_equal(got["status"], st) and np.array_equal(got["score"][good], sc)
                  and np.array_equal(got["best_idx"][good].view(np.uint32), i)
                  and np.array_equal(got["best_dis"][good].view(np.uint32), d1)
                  and np.array_equal(got["cmd"][good].view(np.uint32), cmd))
            return {"templates": T, "matcher": "band" if flags else "greedy", "r": r if flags else None, "k": k, "q": q,
                    "ms_per_step": step_ms,
                    "init_ms": float(np.mean(per[3])), "scan_ms": float(np.mean(per[scan])),
                    "final_ms": float(np.mean(per[5])), "sample_rejected": int(rej.sum()),
                    "sample_cmd_changed": int((cmd != decide(sc)[2]).sum()), "sample_equals_oracle": bool(ok)}

        settings = [(flags, r, k, q) for flags, r in MATCHERS for k, q in rules]
        for s in settings:                                   # warm-up of every setting before any is timed
            run(*s)
        for _ in range(args.rounds):
            for s in settings:
                results.append(run(*s))
    h.set_match(0, 0)
    h.close()
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "batch": B, "steps": args.steps,
            "warmup": args.warmup, "rounds": args.rounds, "sample": n, "tail": len(rows) - n,
            "sample_ok_utterances": int(good.sum()), "results": results}
    print("%4s %-7s %5s %3s %6s %10s %9s %9s %9s %9s %9s %6s" % (
        "T", "matcher", "r", "k", "q", "ms/step", "init ms", "scan ms", "final ms", "rejected", "cmd diff", "oracle"))
    for x in results:
        print("%4d %-7s %5s %3d %6d %10.3f %9.4f %9.3f %9.4f %9d %9d %6s" % (
            x["templates"], x["matcher"], "" if x["r"] is None else x["r"], x["k"], x["q"], x["ms_per_step"], x["init_ms"],
            x["scan_ms"], x["final_ms"], x["sample_rejected"], x["sample_cmd_changed"], x["sample_equals_oracle"]))
    report("bench_rule", info, all(x["sample_equals_oracle"] for x in results), args.json)


if __name__ == "__main__":
    main()
