"""Throughput of the alignment calls (K3p): sr_dtw_path_batch, sr_average_bank, and recognition against an averaged bank,
on BASELINE configs[1]-sized inputs (65 536 one-second utterances of synthetic PCM generated on the device, 20 templates).

  1. sr_dtw_path_batch on 65 536 (utterance, template) pairs at r in {10, 15, 16, 118}: pairs/s and oracle cells/s of the
     kernel alone (tag 7), next to the cells/s of the score-only bank scan (sr_dtw_batch with SR_DTW_BAND, tag 6) at the
     same r; the host call's wall time too (it moves 2 x 187 MB of features and 31 MB of paths).
  2. sr_average_bank at G = 16 384 groups of K = 4 slots (the 65 536 utterances enrolled), iters in {1, 3}: the host
     call's wall time and its kernels' time (tags 7 and 8).
  3. sr_recognise_batch_dev at r = 118 against the 20-slot bank (4 per command) and against its averaged bank (one signed
     slot per command, the others erased): ms per step and the DTW kernel's time (tag 6).

Every row checks a sample against the oracles (tests/oracle_ext/align.c, oracle/sr_oracle.c). The card's name, power limit
and SM clock limit are read in the same run.

    python tools/bench_align.py [--steps 10] [--warmup 2] [--json FILE]
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

import oracle_ext as ox  # noqa: E402
import oracle_bind as ob  # noqa: E402
import sr_b200  # noqa: E402
from bench_match import card  # noqa: E402

U, N_LEN = 8000, 2400
SEED, TPL_SEED = 0x5EED0000, 0x7E3A0000       # bench.py's inputs
NPROC = os.cpu_count() or 1


def timed(h, fn, reps):
    """(wall ms per call, {tag: kernel ms per call}) of fn() repeated reps times"""
    h.timing_enable(64 * reps)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    ker = {}
    for t, ms in h.timing_collect():
        ker[t] = ker.get(t, 0.0) + ms / reps
    h.timing_enable(0)
    return wall, ker, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--templates", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_align: no CUDA device (there is nothing to measure without one)")
    dev = torch.device("cuda:0")
    B, T, n = args.batch, args.templates, args.sample
    h = sr_b200.Handle(0)
    stream = torch.cuda.Stream(dev)
    h.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):                  # features of the utterances and the templates, on the device
        pcm = torch.empty((B, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(pcm.data_ptr(), B, U, SEED, 1, stream.cuda_stream)
        tpl = torch.empty((T, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(tpl.data_ptr(), T, U, TPL_SEED, 1, stream.cuda_stream)
        h.set_bank_dev(0, 0, 4096)
        uftr = torch.zeros((B, 2860), dtype=torch.uint8, device=dev)
        ust = torch.zeros(B, dtype=torch.uint8, device=dev)
        h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, ftr=uftr.data_ptr(), status=ust.data_ptr())
        tftr = torch.zeros((T, 2860), dtype=torch.uint8, device=dev)
        h.recognise_dev(tpl.data_ptr(), U, T, N_LEN, ftr=tftr.data_ptr())
    stream.synchronize()
    h.use_own_stream()
    fin = uftr.cpu().numpy().view(ob.FTR_DTYPE).reshape(B)
    status = ust.cpu().numpy()
    tf = tftr.cpu().numpy().view(ob.FTR_DTYPE).reshape(T)
    bank20 = sr_b200.make_bank(tf)
    results = {"path": [], "average": [], "recognise": []}
    ao, po = ox.align(), ob.port()

    # 1. paths: utterance p against template p % T
    mdl = tf[np.arange(B) % T]
    h.set_bank(bank20, T, 4096)
    for r in (10, 15, 16, 118):
        for _ in range(args.warmup):
            h.dtw_path(fin, mdl, r)
        wall, ker, (dis, path, plen) = timed(h, lambda: h.dtw_path(fin, mdl, r), args.steps)
        wd, wp, wl = ao.dtw_path(fin[:n], mdl[:n], r, nthreads=NPROC)
        ok = bool(np.array_equal(dis[:n], wd) and np.array_equal(path[:n], wp) and np.array_equal(plen[:n], wl))
        cells = sum(po.dtw_batch(fin[p:p + 1], sr_b200.make_bank(mdl[p:p + 1]), 1, 4096, band_r=r)[1] for p in range(n))
        cells_b = cells * B / n
        _, kscan, _ = timed(h, lambda: h.dtw(fin, flags=sr_b200.DTW_BAND, band_r=r, want_best=False), args.steps)
        scan_cells = po.dtw_batch(fin[:n], bank20, T, 4096, band_r=r, nthreads=NPROC)[1] * B / n
        results["path"].append({"r": r, "pairs": B, "kernel_ms": ker[7], "wall_ms": wall, "pairs_per_s": B / (ker[7] * 1e-3),
                                "cells_per_s": cells_b / (ker[7] * 1e-3), "scan_kernel_ms": kscan[6],
                                "scan_cells_per_s": scan_cells / (kscan[6] * 1e-3), "sample_equals_oracle": ok})

    # 2. averaging: the B utterances as G = B / 4 groups of 4 enrolled slots (failed front ends erased)
    K = 4
    G = B // K
    bank = np.full((B, 4096), 0xFF, np.uint8)
    bank[:, :2860] = fin.view(np.uint8).reshape(B, 2860)
    bank[:, 0], bank[:, 1] = 12345 & 0xFF, 12345 >> 8
    bank[status != 0] = 0xFF
    ng = min(G, 64)
    for iters in (1, 3):
        h.average_bank(bank[:4 * K], 4096, K, 118, iters)
        wall, ker, (out, score, anchor) = timed(h, lambda: h.average_bank(bank, 4096, K, 118, iters), max(1, args.steps // 5))
        wo, ws, wa = ao.average_bank(bank[:ng * K], 4096, K, 118, iters, nthreads=NPROC)
        ok = bool(np.array_equal(out[:ng * K], wo) and np.array_equal(score[:ng], ws) and np.array_equal(anchor[:ng], wa))
        results["average"].append({"G": G, "K": K, "r": 118, "iters": iters, "wall_ms": wall, "align_ms": ker.get(7, 0.0),
                                   "update_ms": ker.get(8, 0.0), "sample_equals_oracle": ok})

    # 3. recognition at r = 118 against the 4-per-command bank and against its averaged bank
    avg20, _, _ = h.average_bank(bank20, 4096, K, 118, 3)
    outs = {k: torch.zeros(shape, dtype=dt, device=dev) for k, shape, dt in
            (("score", (B, T), torch.int32), ("best_idx", (B,), torch.int32), ("best_dis", (B,), torch.int32),
             ("cmd", (B,), torch.int32), ("status", (B,), torch.uint8))}
    ptrs = {k: v.data_ptr() for k, v in outs.items()}
    front = ob.recognise_pinned(ob.best_oracle(), sr_b200.synth_pcm_host(n, U, SEED), N_LEN, None, 0, 4096)
    good = front["status"] == 0
    for name, bk in (("4 per command", bank20), ("averaged", avg20)):
        h.set_bank(bk, T, 4096)
        h.set_match(sr_b200.DTW_BAND, 118)
        for _ in range(args.warmup):
            h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs)
        h.sync()
        h.timing_enable(6 * args.steps + 8)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            ev0.record(stream)
            for _ in range(args.steps):
                h.recognise_dev(pcm.data_ptr(), U, B, N_LEN, **ptrs)
            ev1.record(stream)
        stream.synchronize()
        dtw_ms = [ms for t, ms in h.timing_collect() if t == 6]
        h.timing_enable(0)
        h.use_own_stream()
        sc, _ = po.dtw_batch(front["ftr"][good], bk, T, 4096, check_sign=1, band_r=118, nthreads=NPROC)
        got = outs["score"][:n].cpu().numpy().view(np.uint32)
        i = np.argmin(sc, axis=1)
        ok = bool(np.array_equal(got[good], sc) and np.array_equal(outs["best_idx"][:n].cpu().numpy().view(np.uint32)[good], i))
        results["recognise"].append({"bank": name, "signed_slots": int((bk[:, :2].copy().view(np.uint16)[:, 0] == 12345).sum()),
                                     "ms_per_step": ev0.elapsed_time(ev1) / args.steps,
                                     "dtw_ms_mean": float(np.mean(dtw_ms)), "sample_equals_oracle": ok})
    h.set_match(0, 0)

    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "batch": B, "templates": T,
            "steps": args.steps, "sample": n, "results": results}
    c = info["card"]
    print("card: %s, power limit %s, max SM clock %s" % (c.get("name"), c.get("power.limit"), c.get("clocks.max.sm")))
    for x in results["path"]:
        print("path r=%-4d kernel %8.3f ms  wall %8.1f ms  %6.2f Mpairs/s  %6.2f Gcells/s | scan %8.3f ms %6.2f Gcells/s  oracle %s" % (
            x["r"], x["kernel_ms"], x["wall_ms"], x["pairs_per_s"] / 1e6, x["cells_per_s"] / 1e9, x["scan_kernel_ms"],
            x["scan_cells_per_s"] / 1e9, x["sample_equals_oracle"]))
    for x in results["average"]:
        print("average G=%d K=%d iters=%d  wall %8.1f ms  align %8.3f ms  update %7.3f ms  oracle %s" % (
            x["G"], x["K"], x["iters"], x["wall_ms"], x["align_ms"], x["update_ms"], x["sample_equals_oracle"]))
    for x in results["recognise"]:
        print("recognise r=118 %-14s (%2d signed slots)  %8.3f ms/step  dtw %8.3f ms  oracle %s" % (
            x["bank"], x["signed_slots"], x["ms_per_step"], x["dtw_ms_mean"], x["sample_equals_oracle"]))
    print(json.dumps(info))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    h.close()
    if not all(x["sample_equals_oracle"] for v in results.values() for x in v):
        raise SystemExit("bench_align: a sample differs from the oracle")


if __name__ == "__main__":
    main()
