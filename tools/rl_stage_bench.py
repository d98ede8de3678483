#!/usr/bin/env python
"""Read-level network (LatentSpaceLSTM forward) at lstm_size 128 or 384: positions/s and per-stage device times.

    python tools/rl_stage_bench.py [--lstm-size 384] [--windows 0] [--positions 10000] [--reads 50] [--steps 3] [--warmup 1]

Synthetic seeded features (P positions x D reads per window, no empty reads), one device call per step.  Before any
timing, one seeded window (its first 2000 positions) is checked against the torch restatement (oracle/rl_oracle.py):
probabilities within 2e-5, labels identical wherever its top-2 margin exceeds 1e-4.  Prints one JSON line:
`value` = positions / device time per step (CUDA events around every stage on the engine's stream), `e2e` adds the host
copies of the features and probabilities, `stage_ms` = mean device time of each stage over the timed steps.
Default windows: 128 at lstm_size 384 (8 tiles x 2 directions = 16 recurrence clusters of 8 CTAs), 256 at 128 (about
35 GB of scratch at 10 000 positions).  Writes nothing.
"""
import argparse
import json
import os
import statistics
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
    args = ap.parse_args()
    import torch
    from medaka_b200 import libmedaka as lm
    from medaka_b200 import read_level
    from oracle import rl_oracle
    info = lm.require_gpu(0)
    H, P, D = args.lstm_size, args.positions, args.reads
    B = args.windows or (128 if H == 384 else 256)
    sd = rl_oracle.synth_rl_state_dict(0, lstm_size=H)
    x = rl_oracle.synth_rl_features(B, P, D, seed=1, empty_rows=0, ragged=False)
    m = read_level.LatentSpaceLSTM(lstm_size=H)
    m.load_state_dict(sd)
    m.max_cells, m.max_bytes = 1 << 62, 1 << 40     # one device call per step: the stage times cover the whole step
    # correctness first: a seeded sample against the CPU restatement
    xs = np.ascontiguousarray(x[:1, :min(P, 2000)])
    ref = rl_oracle.LatentSpaceLSTM(lstm_size=H)
    ref.load_state_dict(sd)
    ref.eval()
    want = rl_oracle.predict(ref, xs, threads=min(16, os.cpu_count() or 8))
    got = m.forward_arrays(xs)
    err = float(np.abs(got - want).max())
    top2 = np.sort(want, -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > 1e-4
    flips = int((np.argmax(got, -1) != np.argmax(want, -1))[decided].sum())
    if not (err < 2e-5 and flips == 0):
        raise SystemExit("read-level check failed: max |dp| %.3e, label flips %d" % (err, flips))
    m.set_timing(True)
    for _ in range(args.warmup):
        m.forward_arrays(x)
    stages, walls = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        m.forward_arrays(x)
        walls.append(time.perf_counter() - t0)
        stages.append(m.stage_ms())
    mean = {k: statistics.mean(s[k] for s in stages) for k in m.STAGES}
    dev_ms = sum(mean.values())
    print(json.dumps({
        "metric": "read_level_positions_per_s", "model": "LatentSpaceLSTM", "lstm_size": H, "cnn_size": 128,
        "value": B * P / (dev_ms * 1e-3), "unit": "positions/s", "e2e": B * P / statistics.mean(walls),
        "windows": B, "positions": P, "reads": D, "steps": args.steps, "warmup": args.warmup,
        "stage_ms": {k: round(v, 3) for k, v in mean.items()}, "device_ms_per_step": round(dev_ms, 3),
        "check": {"windows": 1, "positions": int(xs.shape[1]), "max_abs_prob_diff": err, "label_flips": flips},
        "gpu": torch.cuda.get_device_name(0), "sm_count": int(info["sm_count"])}))
    m.close()


if __name__ == "__main__":
    main()
