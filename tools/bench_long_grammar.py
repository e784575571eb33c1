"""Throughput of one grammar decode per long recording (include/sr_long_grammar.h, sr_recognise_long_grammar_batch).

Rows: 4 096 synthetic recordings of 30 s under the loop grammar, a 4-word PIN chain and an 11-word chain (position k
restricted to command k mod 5, which keeps its copies within SR_GRAM_COPY_MAX), against a 20-slot bank (5 commands x 4
enrolments) and the averaged bank (sr_average_bank of each command's 4 enrolments); then one recording of 2^27 samples
under the loop grammar. Each row reports the decoder's kernel time (timing tag 13), the call's wall time, decoded frames
per second of decoder time and G cells per second (frames x the summed template lengths of the grammar's copies). Every
row checks the composed oracle (tests/oracle_ext.py) on the first and last recording of every decoder launch and
on random others. The card's name and power limit are read in the same run; the JSON goes to tools/results/.

    python tools/bench_long_grammar.py [--steps 2] [--warmup 1] [--json FILE]
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

GROUP_BYTES = 256 << 20      # kLongGroupBytes: PCM per staged group
REC_BYTES = 256 << 20        # kLongGramRecBytes: records per decoder launch
TAG_LONG_GRAM = 13


def members(bank, T):
    """{slot: frames} of the signed slots of 1..119 frames"""
    out = {}
    for t in range(T):
        sign, n = np.frombuffer(bank[t, :4].tobytes(), np.uint16)
        if sign == sr_b200.SAVE_MASK and 1 <= n <= 119:
            out[t] = int(n)
    return out


def copy_cells(g, mem):
    """sum of the template lengths over the grammar's copies: DP cells per decoded frame"""
    S, _, arcs = g
    return sum(M for s in range(S) for t, M in mem.items() if any(b == s and (m >> (t // 4)) & 1 for _, b, m in arcs))


def launch_edges(B, U, N, S):
    """first and last recording of every decoder launch: per group, consecutive recordings while records fit"""
    G = max(1, min(GROUP_BYTES // (2 * U), B))
    edges = set()
    for g0 in range(0, B, G):
        rows, first = 0, g0
        for b in range(g0, min(g0 + G, B)):
            if rows and (rows + N[b]) * S * 12 > REC_BYTES:
                edges |= {first, b - 1}
                rows, first = 0, b
            rows += N[b]
        edges |= {first, min(g0 + G, B) - 1}
    return edges


def row(h, pcm, bank, T, g, steps, warmup, sample, seed, max_segs=256, max_words=512):
    h.set_bank(bank, T, 4096)
    B, U = pcm.shape
    for _ in range(warmup):
        h.recognise_long_grammar(pcm, g, 1000, max_segs, max_words)
    h.timing_enable(1 << 16)
    h.timing_collect()
    t0 = time.perf_counter()
    for _ in range(steps):
        got = h.recognise_long_grammar(pcm, g, 1000, max_segs, max_words)
    wall = (time.perf_counter() - t0) / steps
    dec_ms = sum(ms for t, ms in h.timing_collect() if t == TAG_LONG_GRAM) / steps
    h.timing_enable(0)
    N = got["frm_num"].sum(axis=1).astype(np.int64)
    assert (got["n_segs"] <= max_segs).all()
    frames = int(N.sum())
    cells = frames * copy_cells(g, members(bank, T))
    rng = np.random.default_rng(seed)
    rows = sorted(launch_edges(B, U, N, g[0]) | set(rng.integers(0, B, sample).tolist()))
    want = ox.recognise_long_grammar(ox.long_oracle(), ob.port(), ox.long_grammar(), np.ascontiguousarray(pcm[rows]), 2400,
                                     bank, T, 4096, g, 1000, max_segs, max_words)
    ok = True
    for i, b in enumerate(rows):
        ok &= int(got["n_words"][b]) == int(want["n_words"][i]) and int(got["total"][b]) == int(want["total"][i])
        m = min(int(want["n_words"][i]), max_words)
        ok &= got["words"][b, :m].tobytes() == want["words"][i, :m].tobytes()
        ok &= int(got["n_segs"][b]) == int(want["n_segs"][i])
    return dict(B=B, U=U, states=g[0], frames=frames, decoder_ms=dec_ms, wall_ms=wall * 1e3,
                frames_per_s=frames / (dec_ms / 1e3), Gcells_per_s=cells / (dec_ms / 1e3) / 1e9,
                words=int(got["n_words"].sum()), oracle_ok=bool(ok), oracle_rows=len(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=8)
    ap.add_argument("--json", default=os.path.join(ROOT, "tools", "results", "bench_long_grammar_h100_700w.json"))
    a = ap.parse_args()
    h = sr_b200.Handle(0)
    tpl = sr_b200.synth_pcm_host(20, 8000, 0x7E3A0000)
    e = ob.port().recognise_batch(tpl, 2400, None, 0, 4096)
    bank20 = sr_b200.make_bank(e["ftr"])
    avg, _, _ = h.average_bank(bank20[:20], 4096, 4, 118, 2)
    grams = {"loop": sr_b200.loop_grammar(), "pin4": sr_b200.chain_grammar(4, 0x1F),
             "chain11": (12, 1 << 11, [(k, k + 1, 1 << (k % 5)) for k in range(11)])}
    res = dict(card=card(), rows={})
    pcm = ox.synth_long(4096, 240000, 0xB30)
    for bname, bank in (("bank20", bank20), ("averaged", avg)):
        for gname, g in grams.items():
            res["rows"]["4096x30s_%s_%s" % (gname, bname)] = row(h, pcm, bank, 20, g, a.steps, a.warmup, a.sample, 0xB31)
    del pcm
    big = ox.synth_long(1, 1 << 27, 0xB40)
    res["rows"]["1x2^27_loop_bank20"] = row(h, big, bank20, 20, grams["loop"], 1, 0, 0, 0xB41, max_segs=1 << 17,
                                             max_words=1 << 19)
    h.close()
    for k, v in res["rows"].items():
        print(k, json.dumps(v))
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(a.json), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    if not all(v["oracle_ok"] for v in res["rows"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
