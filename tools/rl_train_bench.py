"""Read-level training step on the H100: per-stage device times of RLTrainer.train_step (CUDA events inside the
library) and step time (host clock around a step that ends in a synchronise), against torch autograd on the
oracle/rl_oracle.py module in fp32 with RMSprop and clip_grad_norm_, with TF32 allowed and off.

    python tools/rl_train_bench.py [--lstm 128 384] [--P 10000] [--D 100] [--F 5] [--B 100] [--out DIR]

Windows of featuriser-like read-level features (oracle.rl_oracle.featuriser_like_rl_features), random labels.  Every
timed shape runs once untimed first.  Torch runs at B = 1, 2, 4, ... until it runs out of memory; its peak memory is
torch.cuda.max_memory_allocated.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def windows(B, P, D, F, seed=0):
    from oracle import rl_oracle
    x1 = rl_oracle.featuriser_like_rl_features(1, P, D, F=F, seed=seed)
    x = np.repeat(x1, B, axis=0)
    y = np.random.RandomState(seed).randint(0, 5, size=(B, P))
    return x, y


def ours(H, B, P, D, F, steps=1):
    import torch
    from medaka_b200 import training
    from oracle import rl_oracle
    sd = {k: v.numpy() for k, v in rl_oracle.synth_rl_state_dict(0, lstm_size=H, use_dwells=F == 5).items()}
    tr = training.RLTrainer(lstm_size=H, use_dwells=F == 5).load_state_dict(sd)
    x, y = windows(B, P, D, F)
    b = training.TrainBatch(labels=y, read_level_features=x)
    tr.train_step(b, lr=1e-4, max_norm=2.0)                   # warm-up of this shape
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        tr.train_step(b, lr=1e-4, max_norm=2.0)
        t.append(time.perf_counter() - t0)
    out = {"B": B, "step_s": min(t), "stage_ms": tr.stage_ms(),
           "workspace_GB": training.rl_workspace_bytes(H, B, P, D, F)[0] / 1e9}
    tr.close()
    torch.cuda.synchronize()
    return out


def torch_step(H, B, P, D, F, tf32):
    import torch
    from oracle import rl_oracle, rl_train_oracle
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    sd = rl_oracle.synth_rl_state_dict(0, lstm_size=H, use_dwells=F == 5)
    m = rl_train_oracle.build({k: v.numpy() for k, v in sd.items()}, F == 5, dtype=torch.float32).cuda()
    opt = torch.optim.RMSprop(m.parameters(), lr=1e-4, alpha=0.9, eps=1e-7)
    x, y = windows(B, P, D, F)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()

    def step():
        opt.zero_grad()
        loss = torch.nn.CrossEntropyLoss()(rl_train_oracle.logits(m, xt).flatten(0, 1), yt.flatten())
        loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 2.0)
        opt.step()
        torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    step()
    t0 = time.perf_counter()
    step()
    return {"B": B, "step_s": time.perf_counter() - t0, "peak_GB": torch.cuda.max_memory_allocated() / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lstm", type=int, nargs="+", default=[128, 384])
    ap.add_argument("--P", type=int, default=10000)
    ap.add_argument("--D", type=int, default=100)
    ap.add_argument("--F", type=int, default=5)
    ap.add_argument("--B", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rl_train_bench needs a CUDA device")
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip(), "P": a.P, "D": a.D, "F": a.F}
    for H in a.lstm:
        r = {"ours_B%d" % a.B: ours(H, a.B, a.P, a.D, a.F)}
        for tf32 in (True, False):
            fits, b = None, 1
            while b <= a.B:
                try:
                    fits = torch_step(H, b, a.P, a.D, a.F, tf32)
                except torch.cuda.OutOfMemoryError:
                    break
                finally:
                    torch.cuda.empty_cache()
                b *= 2
            r["torch_tf32" if tf32 else "torch_fp32"] = fits
            if fits and tf32:
                r["ours_B%d" % fits["B"]] = ours(H, fits["B"], a.P, a.D, a.F)
        res["lstm%d" % H] = r
        print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rl_train_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
