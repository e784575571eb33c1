"""Recognition time without a decision rule and under the KNN rule SR_DTW_KNN(k), k = 2, 3, 4, under the greedy walk and
the banded DP at r = 10 (sr_set_match), on BASELINE configs[1]'s shape: 65 536 utterances x 1 s (synthetic PCM generated
on the device) against a bank of 20 commands x 4 templates.

Per (matcher, k): W warm-up steps, then K steps of sr_recognise_batch_dev between CUDA events (ms/step), and the
library's own event pairs (sr_timing_*) for best-init (tag 3), the template scan (4 greedy / 6 banded) and the finisher
(tag 5), which under KNN reads the B x 80 per-slot keys. The settings of a matcher alternate, several rounds, after the
warm-up of each. A sample of every row's outputs -- the first utterances of the launch and its last ones -- is checked
against the oracle's composition: its front end (recognise_pinned), its template scan under the same matcher, then the
KNN decision in numpy. The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_knn.py [--steps 20] [--warmup 3] [--rounds 2] [--json FILE]
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
import sr_b200  # noqa: E402
from bench_match import card  # noqa: E402

U, N_LEN = 8000, 2400
SEED, TPL_SEED = 0x5EED0000, 0x7E3A0000       # bench.py's inputs


def knn(sc, k):
    """best_idx and best_dis per row of sc [n][T] under SR_DTW_KNN(k), k = 0: the nearest slot (see tests/test_knn.py)"""
    err = np.uint64(0xFFFFFFFF)
    n, T = sc.shape
    C = (T + 3) // 4
    s = np.full((n, 4 * C), err, np.uint64)
    s[:, :T] = sc
    s = s.reshape(n, C, 4)
    m = np.minimum(max(k, 1), (s != err).sum(axis=2))
    take = np.arange(4)[None, None, :] < m[:, :, None]
    e = np.where(m > 0, np.where(take, np.sort(s, axis=2), 0).sum(axis=2) // np.maximum(m, 1), err).astype(np.uint64)
    slot = np.where(m > 0, np.arange(C)[None, :] * 4 + np.argmin(s, axis=2), 0).astype(np.uint64)
    k1 = ((e << np.uint64(32)) | slot).min(axis=1)
    return (k1 & err).astype(np.uint32), (k1 >> np.uint64(32)).astype(np.uint32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--templates", default="80")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of the settings per matcher")
    ap.add_argument("--sample", type=int, default=256, help="first utterances checked against the oracle")
    ap.add_argument("--tail", type=int, default=32, help="last utterances checked against the oracle")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn: no CUDA device (there is nothing to measure without one)")
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
    band = sr_b200.DTW_BAND
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

        def run(flags, r, k):
            h.set_match(flags | sr_b200.dtw_knn(k), r)
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
            assert all(len(v) == args.steps for v in per.values()), (flags, r, k, {t: len(v) for t, v in per.items()})
            idx = torch.from_numpy(rows).to(dev)
            got = {k: outs[k][idx].cpu().numpy() for k in ("score", "best_idx", "best_dis", "cmd", "status")}
            got["score"] = got["score"].view(np.uint32)
            if (flags, r) not in scores:
                scores[(flags, r)] = ob.port().dtw_batch(front["ftr"][good], bank_h, T, 4096, check_sign=1,
                                                         band_r=r if flags else -1, nthreads=os.cpu_count() or 1)[0]
            sc = scores[(flags, r)]
            i, d1 = knn(sc, k)
            i0, _ = knn(sc, 0)
            ok = (np.array_equal(got["status"], front["status"]) and np.array_equal(got["score"][good], sc)
                  and np.array_equal(got["best_idx"][good].view(np.uint32), i)
                  and np.array_equal(got["best_dis"][good].view(np.uint32), d1)
                  and np.array_equal(got["cmd"][good].view(np.uint32), i // 4))
            return {"templates": T, "matcher": "band" if flags else "greedy", "r": r if flags else None, "k": k,
                    "ms_per_step": ev0.elapsed_time(ev1) / args.steps,
                    "init_ms": float(np.mean(per[3])), "scan_ms": float(np.mean(per[scan])),
                    "final_ms": float(np.mean(per[5])), "sample_cmd_changed": int((i // 4 != i0 // 4).sum()),
                    "sample_equals_oracle": bool(ok)}

        for flags, r in ((0, 0), (band, 10)):
            for k in (0, 2, 3, 4):                           # warm-up of every setting before any is timed
                run(flags, r, k)
            for _ in range(args.rounds):
                for k in (0, 2, 3, 4):
                    results.append(run(flags, r, k))
    h.set_match(0, 0)
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "batch": B, "steps": args.steps,
            "warmup": args.warmup, "rounds": args.rounds, "sample": n, "tail": tail,
            "sample_ok_utterances": int(good.sum()), "results": results}
    print("card: %s, power limit %s, max SM clock %s" % (info["card"].get("name"), info["card"].get("power.limit"),
                                                        info["card"].get("clocks.max.sm")))
    print("%4s %-7s %5s %3s %10s %9s %9s %9s %9s %6s" % ("T", "matcher", "r", "k", "ms/step", "init ms", "scan ms",
                                                         "final ms", "cmd diff", "oracle"))
    for x in results:
        print("%4d %-7s %5s %3d %10.3f %9.4f %9.3f %9.4f %9d %6s" % (
            x["templates"], x["matcher"], "" if x["r"] is None else x["r"], x["k"], x["ms_per_step"], x["init_ms"],
            x["scan_ms"], x["final_ms"], x["sample_cmd_changed"], x["sample_equals_oracle"]))
    print(json.dumps(info))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    h.close()
    if not all(x["sample_equals_oracle"] for x in results):
        raise SystemExit("bench_knn: a sample differs from the oracle")


if __name__ == "__main__":
    main()
