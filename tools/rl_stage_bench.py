#!/usr/bin/env python
"""Read-level network (LatentSpaceLSTM forward) at lstm_size 128 or 384: positions/s and per-stage device times.

    python tools/rl_stage_bench.py [--lstm-size 384] [--windows 0] [--positions 10000] [--reads 50] [--steps 3] [--warmup 1]
                                   [--precision tc[,fp16]] [--dwells]

Synthetic seeded features (P positions x D reads per window, no empty reads), one device call per step; --dwells takes
featuriser-like reads with dwells and a dwell model instead (rl_engine_bench.py's traffic).  --precision names the
engine modes (LatentSpaceLSTM.set_precision): with several, each is warmed up, then the steps alternate between them.
Before any timing, one seeded window (its first 2000 positions) is checked in each mode against the torch restatement
(oracle/rl_oracle.py; the fp16 mode against tests/rl_fp16_oracle.py, fed the engine's LSTM inputs and h): probabilities within 2e-5, labels identical wherever its
top-2 margin exceeds 1e-4.  Prints one JSON line per mode:
`value` = positions / device time per step (CUDA events around every stage on the engine's stream), `e2e` adds the host
copies of the features and probabilities, `stage_ms` = mean device time of each stage over the timed steps.
Default windows: 128 at lstm_size 384 (8 tiles x 2 directions = 16 recurrence clusters of 8 CTAs), 256 at 128 (about
35 GB of scratch at 10 000 positions).  Writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lstm-size", type=int, default=384, choices=[128, 384])
    ap.add_argument("--windows", type=int, default=0, help="0 = 128 at lstm_size 384, 256 at 128")
    ap.add_argument("--positions", type=int, default=10000)
    ap.add_argument("--reads", type=int, default=50)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--precision", default="tc", help="comma-separated modes: tc, fp16")
    ap.add_argument("--dwells", action="store_true")
    args = ap.parse_args()
    modes = args.precision.split(",")
    if not set(modes) <= {"tc", "fp16"}:
        raise SystemExit("--precision: tc and / or fp16")
    import torch
    from medaka_b200 import libmedaka as lm
    from medaka_b200 import read_level
    from oracle import rl_oracle
    from tests import rl_fp16_oracle
    info = lm.require_gpu(0)
    H, P, D = args.lstm_size, args.positions, args.reads
    B = args.windows or (128 if H == 384 else 256)
    sd = rl_oracle.synth_rl_state_dict(0, lstm_size=H, use_dwells=args.dwells)
    if args.dwells:
        x = rl_oracle.featuriser_like_rl_features(B, P, D, F=5, seed=3)
    else:
        x = rl_oracle.synth_rl_features(B, P, D, seed=1, empty_rows=0, ragged=False)
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=args.dwells)
    m.load_state_dict(sd)
    m.max_cells, m.max_bytes = 1 << 62, 1 << 40     # one device call per step: the stage times cover the whole step
    # correctness first: a seeded sample against the CPU restatement
    xs = np.ascontiguousarray(x[:1, :min(P, 2000)])
    ref = rl_oracle.build(sd, use_dwells=args.dwells)
    threads = min(16, os.cpu_count() or 8)
    checks = {}
    for mode in modes:
        m.set_precision(mode)
        got = m.forward_arrays(xs)
        if mode == "fp16":      # the fp16 oracle, its LSTM layers fed the engine's own inputs and h
            feed = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
            want = rl_fp16_oracle.stages(ref, xs, feed=feed, threads=threads)["probs"]
        else:
            want = rl_oracle.predict(ref, xs, threads=threads)
        err = float(np.abs(got - want).max())
        top2 = np.sort(want, -1)[..., -2:]
        decided = (top2[..., 1] - top2[..., 0]) > 1e-4
        flips = int((np.argmax(got, -1) != np.argmax(want, -1))[decided].sum())
        if not (err < 2e-5 and flips == 0):
            raise SystemExit("read-level check failed (%s): max |dp| %.3e, label flips %d" % (mode, err, flips))
        checks[mode] = {"windows": 1, "positions": int(xs.shape[1]), "max_abs_prob_diff": err, "label_flips": flips}
    m.set_timing(True)
    for mode in modes:
        m.set_precision(mode)
        for _ in range(args.warmup):
            m.forward_arrays(x)
    stages, walls = {mode: [] for mode in modes}, {mode: [] for mode in modes}
    for _ in range(args.steps):
        for mode in modes:
            m.set_precision(mode)
            t0 = time.perf_counter()
            m.forward_arrays(x)
            walls[mode].append(time.perf_counter() - t0)
            stages[mode].append(m.stage_ms())
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True).stdout.strip()
    for mode in modes:
        mean = {k: statistics.mean(s[k] for s in stages[mode]) for k in m.STAGES}
        dev_ms = sum(mean.values())
        print(json.dumps({
            "metric": "read_level_positions_per_s", "model": "LatentSpaceLSTM", "lstm_size": H, "cnn_size": 128,
            "precision": mode, "value": B * P / (dev_ms * 1e-3), "unit": "positions/s",
            "e2e": B * P / statistics.mean(walls[mode]), "e2e_steps": [round(B * P / w) for w in walls[mode]],
            "windows": B, "positions": P, "reads": D, "dwells": args.dwells, "steps": args.steps,
            "warmup": args.warmup, "stage_ms": {k: round(v, 3) for k, v in mean.items()},
            "device_ms_per_step": round(dev_ms, 3), "check": checks[mode],
            "gpu": torch.cuda.get_device_name(0), "sm_count": int(info["sm_count"]), "card": card}))
    m.close()


if __name__ == "__main__":
    main()
