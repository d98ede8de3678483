#!/usr/bin/env python
"""Read-level network on reference-shaped traffic: packed asynchronous calls against one synchronous call per batch.

    python tools/rl_engine_bench.py [--lstm-sizes 384,128] [--batches 8] [--batch-size 100] [--positions 10000]
                                    [--reads 100] [--runs 2] [--precision tc[,fp16]]

Traffic: `batches` batches of `batch-size` windows of P positions x D featuriser-like reads with dwells (the reference's
default batch of 100 chunks of 10 000 columns and 100 reads), the same seeded batch every time.  Two ways, alternating in
one process, `runs` times each after one warm-up batch of each:
  packed  LatentSpaceLSTM.predict_async with the look-ahead and reservation run_prediction uses: each call's
          convolution runs when it is submitted, the LSTM once per group of preferred_batch_size() windows
  sync    forward_arrays: the call pattern of the earlier predict_on_batch (mdk_rl_forward calls of windows_per_call
          windows under the default max_cells / max_bytes, each running the recurrences on its own), on this engine, whose
          mdk_rl_forward is submit + wait with one group per call
--precision names the engine modes (LatentSpaceLSTM.set_precision); with several, every mode is warmed up and each run
goes through the modes in turn, both ways each.
Prints one JSON line per lstm_size and mode: positions/s of every run (host clock from the first submit to the last result in
host memory), the max |dprob| and the label mismatches between the two ways on the batch, and the card's name, power
limit and max SM clock read in the same call.  Writes nothing.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Batch(object):
    def __init__(self, x):
        self.read_level_features = x


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _packed(m, batch, n, P):
    """run_prediction's look-ahead loop (prediction.py) over n copies of the batch; returns (seconds, first result)."""
    B = len(batch.read_level_features)
    depth = m.lookahead(B, P)
    m.reserve(max(m.preferred_batch_size(), B), P)
    pending, first = collections.deque(), None
    t0 = time.perf_counter()
    for _ in range(n):
        while len(pending) >= depth:
            h = pending.popleft()
            p = h.result()
            first = (p.numpy(), h.labels) if first is None else first
        pending.append(m.predict_async(batch, slots=depth + 1))
    while pending:
        h = pending.popleft()
        p = h.result()
        first = (p.numpy(), h.labels) if first is None else first
    return time.perf_counter() - t0, first


def _sync(m, batch, n):
    t0 = time.perf_counter()
    first = None
    for _ in range(n):
        p = m.forward_arrays(batch.read_level_features)
        first = p if first is None else first
    return time.perf_counter() - t0, first


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lstm-sizes", default="384,128")
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--batch-size", type=int, default=100)
    ap.add_argument("--positions", type=int, default=10000)
    ap.add_argument("--reads", type=int, default=100)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--precision", default="tc", help="comma-separated modes: tc, fp16")
    args = ap.parse_args()
    modes = args.precision.split(",")
    if not set(modes) <= {"tc", "fp16"}:
        raise SystemExit("--precision: tc and / or fp16")
    from medaka_b200 import libmedaka as lm
    from medaka_b200 import read_level
    from oracle import rl_oracle
    lm.require_gpu(0)
    B, P, D, n = args.batch_size, args.positions, args.reads, args.batches
    batch = _Batch(rl_oracle.featuriser_like_rl_features(B, P, D, F=5, seed=3))
    for H in (int(h) for h in args.lstm_sizes.split(",")):
        m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=True)
        m.load_state_dict(rl_oracle.synth_rl_state_dict(0, lstm_size=H, use_dwells=True))
        for mode in modes:                               # warm-up: every kernel and buffer of both ways
            m.set_precision(mode)
            _packed(m, batch, 1, P)
            _sync(m, batch, 1)
        rates = {mode: {"packed": [], "sync": []} for mode in modes}
        firsts = {mode: {} for mode in modes}
        card = _card()
        for _ in range(args.runs):
            for mode in modes:
                m.set_precision(mode)
                dt, firsts[mode]["packed"] = _packed(m, batch, n, P)
                rates[mode]["packed"].append(n * B * P / dt)
                dt, firsts[mode]["sync"] = _sync(m, batch, n)
                rates[mode]["sync"].append(n * B * P / dt)
        card_after = _card()
        for mode in modes:
            pp, pl = firsts[mode]["packed"]
            ps = firsts[mode]["sync"]
            r = rates[mode]
            print(json.dumps({
                "metric": "read_level_positions_per_s", "lstm_size": H, "precision": mode, "batches": n,
                "batch_size": B, "positions": P, "reads": D, "dwells": True, "group_windows": m.preferred_batch_size(),
                "sync_windows_per_call": m.windows_per_call(P, D, 5),
                "packed": [round(v) for v in r["packed"]], "sync": [round(v) for v in r["sync"]],
                "speedup": round(min(r["packed"]) / max(r["sync"]), 3),
                "max_abs_prob_diff": float(np.abs(pp - ps).max()),
                "label_mismatches_packed_vs_sync_argmax": int((pl != np.argmax(ps, -1)).sum()),
                "bit_identical": bool(np.array_equal(pp, ps)),
                **card, "card_after": card_after}))
        m.close()


if __name__ == "__main__":
    main()
