#!/usr/bin/env python
"""Consensus GRU at gru_size 256 (the width `medaka train` builds by default) against 128, in one process.

    python tools/gru256_bench.py [--cols 10000] [--groups 3] [--warmup 1] [--precision tc,fp16] [--rounds 1]

For each width: a model with seeded synthetic weights (F = 10), one engine group of preferred_batch_size() windows (one
wave of that width's recurrence) x --cols featuriser-like columns, resident on the device, run --warmup times and then
--groups times through mdk_engine_forward_dev.  The timed region spans the groups (mdk_engine_timer_start / _stop,
device events).  Prints one JSON line per width: positions / s, the per-stage means of mdk_engine_mean_timings over the
timed groups, the GRU multiply-accumulates per position, and the card's name and power limit.  With several --precision
modes (GRUModel.set_precision: tc, fp16, fp32) each width runs in each mode in turn, --rounds times over.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True)
    name, limit = [s.strip() for s in out.stdout.strip().split(",")[:2]] if out.returncode == 0 else (None, None)
    return {"name": name, "power_limit_w": float(limit) if limit else None}


def gru_macs_per_position(H, F=10):
    """Multiply-accumulates of the two bidirectional GRU layers per position (input projections and recurrences)."""
    return 2 * (3 * H * F + 3 * H * H) + 2 * (3 * H * 2 * H + 3 * H * H)


def run(H, feats_all, cols, groups, warmup, precision="tc"):
    import torch
    from medaka_b200 import libmedaka as lm, models
    from oracle import synth
    lib, ffi = lm.lib, lm.ffi
    m = models.GRUModel(num_features=10, gru_size=H)
    try:
        m.load_state_dict(synth.synth_state_dict(0, gru_size=H))
        m.set_precision(precision)
        B = m.preferred_batch_size()
        x = torch.from_numpy(feats_all[:B]).cuda()
        probs = torch.empty((B, cols, 5), dtype=torch.float32, device="cuda")
        labels = torch.empty((B, cols), dtype=torch.uint8, device="cuda")
        m.reserve(B, cols)
        torch.cuda.synchronize()

        def forward():
            lm.check(lib.mdk_engine_forward_dev(m.engine, ffi.cast("const float *", x.data_ptr()), B, cols,
                                                ffi.cast("float *", probs.data_ptr()), ffi.NULL,
                                                ffi.cast("uint8_t *", labels.data_ptr())))

        for _ in range(warmup):
            forward()
        lm.check(lib.mdk_engine_sync(m.engine))
        lm.check(lib.mdk_engine_timer_start(m.engine))
        for _ in range(groups):
            forward()
        ms = ffi.new("float *")
        lm.check(lib.mdk_engine_timer_stop(m.engine, ms))
        t = ffi.new("mdk_timings *")
        lm.check(lib.mdk_engine_mean_timings(m.engine, groups, t))
        stages = {k: round(float(getattr(t, k)), 3) for k in ("inproj0_ms", "rec0_ms", "inproj1_ms", "rec1_ms",
                                                                "head_ms", "total_ms")}
        pos = groups * B * cols
        return {"gru_size": H, "precision": precision, "windows_per_group": B, "cols": cols, "groups": groups,
                "positions_per_s": pos / (ms[0] / 1e3), "elapsed_ms": float(ms[0]), "stage_ms_mean": stages,
                "gru_macs_per_position": gru_macs_per_position(H)}
    finally:
        m.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=10000)
    ap.add_argument("--groups", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--precision", default="tc", help="comma-separated engine modes, run alternately")
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    from medaka_b200 import libmedaka as lm, models
    from oracle import gru_oracle
    lm.require_gpu(0)
    m = models.GRUModel(num_features=10)
    most = m.preferred_batch_size()      # the 128 engine's wave is the larger one
    m.close()
    feats = np.ascontiguousarray(gru_oracle.featuriser_like_features(most, args.cols, 10, seed=3))
    info = card()
    for _ in range(args.rounds):
        for H in (256, 128):
            for mode in args.precision.split(","):
                r = run(H, feats, args.cols, args.groups, args.warmup, mode)
                r.update(card=info["name"], power_limit_w=info["power_limit_w"], timing="device events")
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
