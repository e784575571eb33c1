"""Recognition time under each template matcher: the reference's greedy walk, the banded DP with and without the 2:1
length guard (SR_DTW_ANY_RATE) and the symmetric P = 1 DP (sr_set_match) at several radii, on BASELINE configs[1]'s shape (65 536 utterances x 1 s, 20 templates, synthetic PCM
generated on the device).

Per matcher: W warm-up steps, then K steps of sr_recognise_batch_dev between CUDA events (ms/step), the DTW kernel's own
time from the library's event pairs (sr_timing_*, tag 4 greedy / 6 banded / 14 symmetric), and lattice cells per second =
the cells the banded oracle evaluates at the same radius on a sample of utterances, scaled to the batch, over the DTW kernel
time. r = 15 and r = 16 sit on either side of the kernel choice (warp-scan form / whole-row form) and are run alternately,
several rounds; the symmetric rows and the banded rows without the guard at r = 10, 16 and 118 alternate with the banded
rows at the same radii. The cells of those rows are the guarded banded DP's, so their cells per second compare the same
work. The lifter rows (SR_DTW_LIFTER) run the greedy walk, the banded DP at r = 10 and 16, the banded DP without the guard
at r = 118 and the symmetric DP at r = 10 with the bit off and on, alternately, several rounds; they do the same DP work,
so their difference is the cost of liftering each staged row. --rows lifter runs those rows alone. A sample of every
matcher's outputs -- the first utterances of the launch and its last ones -- is checked against the oracle's own
composition: its front end (recognise_pinned), its template scan under the same matcher (oracle_ext/sym.c for the symmetric DP,
oracle_ext/rate.c for the banded DP without the guard, under SR_DTW_LIFTER on liftered rows: tests/lifter_ref.py),
the strict '<' first-wins argmin. The card's name, power limit and SM clock limit are read in the same run.

    python tools/bench_match.py [--steps 20] [--warmup 3] [--rounds 3] [--rows all|lifter] [--json FILE]
"""
import argparse

import numpy as np
import torch

# benchlib first: it puts the package and tests/ on sys.path
from benchlib import N_LEN, NPROC, SEED, U, card, cuda_device, device_bank, event_steps, report, sample_rows
import lifter_ref
import oracle_bind as ob
import sr_b200


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--templates", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of r = 15 and r = 16")
    ap.add_argument("--sample", type=int, default=256, help="first utterances checked against the oracle")
    ap.add_argument("--tail", type=int, default=32, help="last utterances checked against the oracle")
    ap.add_argument("--rows", choices=("all", "lifter"), default="all", help="every matcher's rows, or the lifter rows alone")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()

    dev = cuda_device("bench_match")
    B, T, n = args.batch, args.templates, min(args.sample, args.batch)
    stream = torch.cuda.Stream(dev)
    h = sr_b200.Handle(0)
    h.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        pcm = torch.empty((B, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(pcm.data_ptr(), B, U, SEED, 1, stream.cuda_stream)
    bank = device_bank(h, stream, T)
    with torch.cuda.stream(stream):
        outs = {k: torch.zeros(shape, dtype=dt, device=dev) for k, shape, dt in
                (("seg_off", (B, 6), torch.int32), ("ftr", (B, 2860), torch.uint8), ("score", (B, T), torch.int32),
                 ("best_idx", (B,), torch.int32), ("best_dis", (B,), torch.int32), ("cmd", (B,), torch.int32),
                 ("status", (B,), torch.uint8))}
    ptrs = {k: v.data_ptr() for k, v in outs.items()}

    # the oracle's composition on the sample (the first n utterances and the last `tail`): the front end once, the
    # template scan per matcher
    bank_h = bank.cpu().numpy()
    rows = sample_rows(B, n, args.tail)
    sample_pcm = pcm[torch.from_numpy(rows).to(dev)].cpu().numpy().view(np.uint16)
    front = ob.recognise_pinned(ob.best_oracle(), sample_pcm, N_LEN, None, 0, 4096)
    good = front["status"] == 0
    SYM = sr_b200.DTW_SYM_P1
    RATE = sr_b200.DTW_BAND | sr_b200.DTW_ANY_RATE
    LIFT = sr_b200.DTW_LIFTER

    def oracle(flags, r):
        """the matcher's scores, and the cells of the port's greedy or banded DP at the same radius"""
        _, cells = ob.port().dtw_batch(front["ftr"][good], bank_h, T, 4096, check_sign=1, band_r=r if flags & ~LIFT else -1,
                                       nthreads=NPROC)
        return lifter_ref.match_scores(front["ftr"][good], bank_h, T, flags, r), cells

    def run(flags, r):
        h.set_match(flags, r)
        step_ms, recs = event_steps(h, stream, lambda: h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs), args.steps,
                                    args.warmup, 6 * args.steps + 8)
        tag = 14 if flags & SYM else 6 if flags & sr_b200.DTW_BAND else 4
        dtw_ms = [ms for t, ms in recs if t == tag]
        assert len(dtw_ms) == args.steps, (flags, r, len(dtw_ms))
        # outputs of the last step against the oracle on the sample
        idx = torch.from_numpy(rows).to(dev)
        got = {k: outs[k][idx].cpu().numpy() for k in ("score", "best_idx", "best_dis", "cmd", "status")}
        got["score"] = got["score"].view(np.uint32)
        sc, cells = oracle(flags, r)
        i = np.argmin(sc, axis=1)
        ok = (np.array_equal(got["status"], front["status"]) and np.array_equal(got["score"][good], sc)
              and np.array_equal(got["best_idx"][good].view(np.uint32), i)
              and np.array_equal(got["best_dis"][good].view(np.uint32), sc[np.arange(len(i)), i])
              and np.array_equal(got["cmd"][good].view(np.uint32), i // 4))
        cells_batch = cells * B / len(rows)
        m = flags & ~LIFT
        name = ("greedy" if not m else "sym" if m == SYM else "band-any" if m == RATE else "band") + ("+lift" if flags & LIFT else "")
        return {"matcher": name, "r": r if m else None,
                "ms_per_step": step_ms,
                "dtw_ms_mean": float(np.mean(dtw_ms)), "dtw_ms_min": float(np.min(dtw_ms)), "dtw_ms_max": float(np.max(dtw_ms)),
                "oracle_cells_per_step": cells_batch, "cells_per_s": cells_batch / (float(np.mean(dtw_ms)) * 1e-3),
                "sample_equals_oracle": bool(ok)}

    band = sr_b200.DTW_BAND
    plan = [(0, 0), (band, 10)] + [(band, r) for _ in range(args.rounds) for r in (15, 16)] + [(band, 32), (band, 118), (0, 0)]
    plan += [(f, r) for _ in range(args.rounds) for r in (10, 16, 118) for f in (band, SYM, RATE)]
    lifter_plan = [(f | lift, r) for _ in range(args.rounds) for f, r in ((0, 0), (band, 10), (band, 16), (RATE, 118), (SYM, 10))
                   for lift in (0, LIFT)]
    plan = lifter_plan if args.rows == "lifter" else plan + lifter_plan
    results = [run(f, r) for f, r in plan]
    h.set_match(0, 0)
    h.close()
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "batch": B, "templates": T,
            "steps": args.steps, "warmup": args.warmup, "sample": n, "tail": len(rows) - n,
            "sample_ok_utterances": int(good.sum()), "results": results}
    print("%-14s %5s %10s %12s %22s %10s %6s" % ("matcher", "r", "ms/step", "dtw ms mean", "dtw ms min-max", "Gcells/s", "oracle"))
    for x in results:
        print("%-14s %5s %10.3f %12.3f %10.3f-%-11.3f %10.2f %6s" % (
            x["matcher"], "" if x["r"] is None else x["r"], x["ms_per_step"], x["dtw_ms_mean"], x["dtw_ms_min"],
            x["dtw_ms_max"], x["cells_per_s"] / 1e9, x["sample_equals_oracle"]))
    report("bench_match", info, all(x["sample_equals_oracle"] for x in results), args.json)


if __name__ == "__main__":
    main()
