#!/usr/bin/env python
"""Recurrent kernels of the tensor-core path at one and two 16-window tiles per CTA, on a full and on a half GPU.

    python tools/rec_wave_bench.py [--cols 10000] [--repeats 4] [--precision tc,fp16]

Three device-resident forwards of the same 2112 x cols / 2 positions, run alternately `--repeats` times after one
warm-up each (seeded synthetic weights and features, F = 10):
  one  1056 windows x cols      one tile per CTA, 132 CTAs (the engine's default group)
  two  2112 windows x cols / 2  two tiles per CTA, 132 CTAs (every SM busy with the two-tile kernel)
  half 1056 windows x cols      two tiles per CTA, 66 CTAs (half of the SMs idle)
With several --precision modes (GRUModel.set_precision: tc, fp16, fp32) every case runs in each, alternating within a
repeat.  Per forward: positions / s and the per-stage times from the engine's stage events (mdk_engine_mean_timings),
and the median SM clock sampled through NVML while it ran.  Prints one JSON line with the card, its power limit, every
run and the medians.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Clock(object):
    """Median SM clock (MHz) over a block of work, sampled every 5 ms through NVML; None without pynvml."""

    def __init__(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(0)
        except Exception:
            self.nv = None

    def card(self):
        if self.nv is None:
            return {"name": None, "power_limit_w": None, "sm_max_mhz": None}
        name = self.nv.nvmlDeviceGetName(self.h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": self.nv.nvmlDeviceGetEnforcedPowerLimit(self.h) / 1000.0,
                "sm_max_mhz": self.nv.nvmlDeviceGetMaxClockInfo(self.h, self.nv.NVML_CLOCK_SM)}

    def during(self, fn):
        if self.nv is None:
            fn()
            return None
        samples, stop = [], []

        def poll():
            while not stop:
                samples.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
                time.sleep(0.005)
        th = threading.Thread(target=poll)
        th.start()
        try:
            fn()
        finally:
            stop.append(True)
            th.join()
        return statistics.median(samples) if samples else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=4)
    ap.add_argument("--precision", default="tc", help="comma-separated engine modes, run alternately")
    args = ap.parse_args()
    modes = args.precision.split(",")
    from medaka_b200 import libmedaka as lm
    from medaka_b200 import models
    from oracle import synth
    lib, ffi = lm.load(), lm.ffi
    info = lm.require_gpu(0)
    sms = int(info["sm_count"])
    T = args.cols - args.cols % 2
    B1 = 8 * sms                                  # one CTA per (tile, direction) at one tile per CTA
    shapes = {"one": ("one", B1, T), "two": ("pp", 2 * B1, T // 2), "half": ("pp", B1, T)}
    cases = {(k if len(modes) == 1 else "%s/%s" % (p, k)): (p,) + c for p in modes for k, c in shapes.items()}
    m = models.GRUModel(num_features=10)
    m.load_state_dict(synth.synth_state_dict(0))
    m.reserve(B1, T)
    P = B1 * T

    def dalloc(nbytes):
        pp = ffi.new("void **")
        lm.check(lib.mdk_dev_alloc(0, nbytes, pp))
        return pp[0]
    d_feats, d_probs, d_labels = dalloc(P * 10 * 4), dalloc(P * 5 * 4), dalloc(P)
    x = synth.synth_features_fast(B1, T, 10, seed=1)
    lm.check(lib.mdk_memcpy_h2d(0, d_feats, ffi.from_buffer(x), x.nbytes))
    tm = ffi.new("mdk_timings *")
    clock = Clock()

    STAGES = ("inproj0_ms", "rec0_ms", "inproj1_ms", "rec1_ms", "head_ms", "total_ms")

    def forward(precision, mode, B, cols):
        m.set_precision(precision)
        m.set_rec_mode(mode)

        def run():
            lm.check(lib.mdk_engine_forward_dev(m.engine, ffi.cast("const float *", d_feats), B, cols,
                                                ffi.cast("float *", d_probs), ffi.NULL, ffi.cast("uint8_t *", d_labels)))
            lm.check(lib.mdk_engine_sync(m.engine))
        mhz = clock.during(run)
        lm.check(lib.mdk_engine_mean_timings(m.engine, 1, tm))
        r = {k: float(getattr(tm, k)) for k in STAGES}
        r.update(positions_per_s=B * cols / (r["total_ms"] / 1e3), sm_mhz=mhz)
        return r

    for c in cases.values():
        forward(*c)
    runs = {k: [] for k in cases}
    for _ in range(args.repeats):
        for k, c in cases.items():
            runs[k].append(forward(*c))
    med = {k: {f: statistics.median(r[f] for r in v) if v[0][f] is not None else None
               for f in STAGES + ("positions_per_s", "sm_mhz")} for k, v in runs.items()}
    print(json.dumps({
        "card": clock.card(), "sm_count": sms, "positions": P, "repeats": args.repeats,
        "cases": {k: {"precision": c[0], "rec_mode": c[1], "windows": c[2], "cols": c[3]} for k, c in cases.items()},
        "median": med, "runs": runs}))
    m.close()


if __name__ == "__main__":
    main()
