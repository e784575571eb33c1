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
from bench_match import card  # noqa: E402
from refs import decide  # noqa: E402

U, N_LEN = 8000, 2400
SEED, TPL_SEED = 0x5EED0000, 0x7E3A0000       # bench.py's inputs
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

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rule: no CUDA device (there is nothing to measure without one)")
    dev = torch.device("cuda:0")
    B, n = args.batch, min(args.sample, args.batch)
    stream = torch.cuda.Stream(dev)
    h = sr_b200.Handle(0)
    h.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        pcm = torch.empty((B, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(pcm.data_ptr(), B, U, SEED, 1, stream.cuda_stream)
    tail = min(args.tail, B - n)
    rows = np.concatenate([np.arange(n), np.arange(B - tail, B)])
    stream.synchronize()
    sample_pcm = pcm[torch.from_numpy(rows).to(dev)].cpu().numpy().view(np.uint16)
    front = ob.recognise_pinned(ob.best_oracle(), sample_pcm, N_LEN, None, 0, 4096)
    good = front["status"] == 0
    results = []
    for T in [int(x) for x in args.templates.split(",")]:
        with torch.cuda.stream(stream):
            tpl = torch.empty((T, U), dtype=torch.int16, device=dev)
            sr_b200.synth_pcm_dev(tpl.data_ptr(), T, U, TPL_SEED, 1, stream.cuda_stream)
            tftr = torch.zeros((T, 2860), dtype=torch.uint8, device=dev)
            h.set_bank_dev(0, 0, 4096)
            h.recognise_dev(tpl.data_ptr(), U, T, N_LEN, ftr=tftr.data_ptr())
            bank = torch.full((T, 4096), 255, dtype=torch.uint8, device=dev)
            bank[:, :2860] = tftr
            bank[:, 0], bank[:, 1] = 12345 & 0xFF, 12345 >> 8
            outs = {k: torch.zeros(shape, dtype=dt, device=dev) for k, shape, dt in
                    (("seg_off", (B, 6), torch.int32), ("ftr", (B, 2860), torch.uint8), ("score", (B, T), torch.int32),
                     ("best_idx", (B,), torch.int32), ("best_dis", (B,), torch.int32), ("cmd", (B,), torch.int32),
                     ("status", (B,), torch.uint8))}
        stream.synchronize()
        h.set_bank_dev(bank.data_ptr(), T, 4096)
        ptrs = {k: v.data_ptr() for k, v in outs.items()}
        bank_h = bank.cpu().numpy()
        scores = {}

        def run(flags, r, k, q):
            h.set_match(flags | sr_b200.dtw_knn(k) | sr_b200.dtw_reject(q), r)
            with torch.cuda.stream(stream):
                for _ in range(args.warmup):
                    h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs)
            stream.synchronize()
            h.timing_enable(6 * args.steps + 8)
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                ev0.record(stream)
                for _ in range(args.steps):
                    h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs)
                ev1.record(stream)
            stream.synchronize()
            recs = h.timing_collect()
            h.timing_enable(0)
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
                    "ms_per_step": ev0.elapsed_time(ev1) / args.steps,
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
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "batch": B, "steps": args.steps,
            "warmup": args.warmup, "rounds": args.rounds, "sample": n, "tail": tail,
            "sample_ok_utterances": int(good.sum()), "results": results}
    print("card: %s, power limit %s, max SM clock %s" % (info["card"].get("name"), info["card"].get("power.limit"),
                                                        info["card"].get("clocks.max.sm")))
    print("%4s %-7s %5s %3s %6s %10s %9s %9s %9s %9s %9s %6s" % (
        "T", "matcher", "r", "k", "q", "ms/step", "init ms", "scan ms", "final ms", "rejected", "cmd diff", "oracle"))
    for x in results:
        print("%4d %-7s %5s %3d %6d %10.3f %9.4f %9.3f %9.4f %9d %9d %6s" % (
            x["templates"], x["matcher"], "" if x["r"] is None else x["r"], x["k"], x["q"], x["ms_per_step"], x["init_ms"],
            x["scan_ms"], x["final_ms"], x["sample_rejected"], x["sample_cmd_changed"], x["sample_equals_oracle"]))
    print(json.dumps(info))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    h.close()
    if not all(x["sample_equals_oracle"] for x in results):
        raise SystemExit("bench_rule: a sample differs from the oracle")


if __name__ == "__main__":
    main()
