"""What the benchmark tools in tools/ share, so that no tool imports another: the card a run measured, the device
check, the two timing windows (a host clock, and CUDA events around recognition steps), bench.py's recognition inputs
and their template bank, the rows checked against the oracle, the launch edges of the connected-word calls, and the
report every tool ends with. Importing it puts the package and tests/ on sys.path.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "stm32-speech-recognition_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_bind as ob  # noqa: E402
import sr_b200  # noqa: E402
from refs import piece_plan, pieces, seq_launches  # noqa: E402

U, N_LEN = 8000, 2400
SEED, TPL_SEED = 0x5EED0000, 0x7E3A0000       # bench.py's inputs
HBM_PEAK = 3.35e12                             # bytes/s, H100 SXM data sheet
NPROC = os.cpu_count() or 1


def card():
    """name, power limit and max SM clock of GPU 0, as nvidia-smi reports them (read only)"""
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def cuda_device(tool):
    """cuda:0, or exit naming the tool when there is no CUDA device"""
    if not torch.cuda.is_available():
        raise SystemExit("%s: no CUDA device (there is nothing to measure without one)" % tool)
    return torch.device("cuda:0")


def timed(h, fn, reps, cap):
    """(wall ms per call, the library's timing records [(tag, ms), ...], last result) of fn() repeated reps times, on a
    host clock that starts on an idle stream and stops after the handle's stream has synchronised; cap is the number
    of timing records the window may hold"""
    h.timing_enable(cap)
    h.timing_collect()                        # drains records from before the window, once queued work has finished
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    h.sync()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    recs = h.timing_collect()
    h.timing_enable(0)
    return wall, recs, out


def per_call(recs, reps):
    """{tag: kernel ms per call} of the timing records of reps calls"""
    ker = {}
    for t, ms in recs:
        ker[t] = ker.get(t, 0.0) + ms / reps
    return ker


def event_steps(h, stream, step, steps, warmup, cap=0):
    """(ms per step, the library's timing records [(tag, ms), ...]) of `steps` calls of step() between CUDA events on
    stream, after `warmup` calls. With a handle, the warm-up is waited for before the window and the window holds
    up to cap timing records; h is None for a call without one, which records nothing."""
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            step()
    if h is not None:
        stream.synchronize()
        h.timing_enable(cap)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        ev0.record(stream)
        for _ in range(steps):
            step()
        ev1.record(stream)
    stream.synchronize()
    recs = []
    if h is not None:
        recs = h.timing_collect()
        h.timing_enable(0)
    return ev0.elapsed_time(ev1) / steps, recs


def device_bank(h, stream, T):
    """the bank of T templates synthesised on the device from TPL_SEED, recognised by h into 4096-byte slots signed
    with save_sign 12345, and set as h's bank in place: the caller keeps the returned tensor alive"""
    dev = torch.device("cuda:0")
    with torch.cuda.stream(stream):
        tpl = torch.empty((T, U), dtype=torch.int16, device=dev)
        sr_b200.synth_pcm_dev(tpl.data_ptr(), T, U, TPL_SEED, 1, stream.cuda_stream)
        tftr = torch.zeros((T, 2860), dtype=torch.uint8, device=dev)
        h.set_bank_dev(0, 0, 4096)
        h.recognise_dev(tpl.data_ptr(), U, T, N_LEN, ftr=tftr.data_ptr())
        bank = torch.full((T, 4096), 255, dtype=torch.uint8, device=dev)
        bank[:, :2860] = tftr
        bank[:, 0], bank[:, 1] = 12345 & 0xFF, 12345 >> 8
    stream.synchronize()
    h.set_bank_dev(bank.data_ptr(), T, 4096)
    return bank


def sample_rows(B, n, tail):
    """the utterances of a launch of B checked against the oracle: the first n and the last `tail` of the others"""
    return np.concatenate([np.arange(n), np.arange(B - min(tail, B - n), B)])


def edges(ranges):
    """the first and last index of every range [lo, hi)"""
    return {i for lo, hi in ranges for i in (lo, hi - 1)}


def e2e_edges(frm_num, seq_ranges=None):
    """the captures holding the first and last get_mfcc piece of every piece launch and, given the decoder's launch ranges
    over the captures' segments with frames (default: one sequence per segment, K6), of every decoder launch"""
    B = len(frm_num)
    e = piece_plan(pieces(frm_num).sum(1))[1]
    if seq_ranges is None:
        owner = np.repeat(np.arange(B), (frm_num > 0).sum(1))
        e |= {int(owner[i]) for i in edges(seq_launches([0, len(owner)]))}
    else:
        e |= edges(seq_ranges)
    return e


def synth_bank(T, seed):
    """a host bank of T synthetic templates of 50..100 frames"""
    ftr = sr_b200.synth_ftr_host(T, seed, 50, 100).view(ob.FTR_DTYPE).reshape(T)
    return sr_b200.make_bank(ftr)


def report(tool, info, ok, json_path):
    """print the card line and info as one JSON line, write info to json_path when one is given, and exit non-zero
    when ok is false (a sample differs from the oracle)"""
    c = info["card"]
    print("card: %s, power limit %s, max SM clock %s" % (c.get("name"), c.get("power.limit"), c.get("clocks.max.sm")))
    print(json.dumps(info))
    if json_path:
        os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
        with open(json_path, "w") as f:
            json.dump(info, f, indent=1)
    if not ok:
        raise SystemExit("%s: a sample differs from the oracle" % tool)
