"""Training step on the H100: this package's GRUTrainer.train_step against torch's own fp32 training step on the same
data and GPU, at the reference's default training shape (100 windows x 10 000 columns, `medaka train --batch_size 100`).

  ours   forward (saved activations), loss, BPTT, reductions, clip, RMSprop, weight repack: medaka_b200/csrc/gru_train.cu;
         a per-stage split from CUDA events (GRUTrainer.stage_ms) and the BPTT kernel at the chosen windows per CTA
         against 8 per CTA
  torch  nn.GRU + nn.Linear + CrossEntropyLoss + clip_grad_norm_ + RMSprop (the reference's run_epoch step without
         GradScaler, which is a no-op scale at fp32), cuDNN with TF32 allowed (torch's default) and with TF32 off

Prints one JSON line per measurement and the card's name and power limit, read in the same call.
    python tools/train_bench.py [--steps 5] [--warmup 2] [--B 100] [--T 10000] [--out DIR]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ours(sd, x, y, H, steps, warmup, nb=0):
    from medaka_b200 import training
    tr = training.GRUTrainer(num_features=x.shape[2], gru_size=H)
    tr.load_state_dict(sd)
    tr.set_bptt_windows(nb)
    for _ in range(warmup):
        tr.train_step((x, y), lr=1e-4, max_norm=2.0)
    stages = {}
    t0 = time.perf_counter()
    for _ in range(steps):
        loss, _, norm, _ = tr.train_step((x, y), lr=1e-4, max_norm=2.0)
        for k, v in tr.stage_ms().items():
            stages[k] = stages.get(k, 0.0) + v / steps
    dt = (time.perf_counter() - t0) / steps
    tr.close()
    return dt, stages, loss


def torch_step(sd, x, y, H, steps, warmup, tf32):
    import torch
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    dev = torch.device("cuda")
    gru = torch.nn.GRU(x.shape[2], H, num_layers=2, bidirectional=True, batch_first=True).to(dev)
    lin = torch.nn.Linear(2 * H, 5).to(dev)
    gru.load_state_dict({k[4:]: torch.from_numpy(v) for k, v in sd.items() if k.startswith("gru.")})
    lin.load_state_dict({k[7:]: torch.from_numpy(v) for k, v in sd.items() if k.startswith("linear.")})
    params = list(gru.parameters()) + list(lin.parameters())
    opt = torch.optim.RMSprop(params, lr=1e-4, alpha=0.9, eps=1e-7, momentum=0.0)
    loss_fn = torch.nn.CrossEntropyLoss()
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y.astype(np.int64)).to(dev)

    def step():
        opt.zero_grad()
        logits = lin(gru(xt)[0])
        loss = loss_fn(logits.flatten(0, 1), yt.flatten())
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, max_norm=2.0)
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        loss = step()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    out = float(loss.item())
    del gru, lin, opt, xt, yt
    torch.cuda.empty_cache()
    return dt, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--B", type=int, default=100)
    ap.add_argument("--T", type=int, default=10000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from oracle import synth
    gpu = card()
    print(json.dumps({"card": gpu}), flush=True)
    results = []
    F = 10
    x = synth.synth_features_fast(a.B, a.T, F, seed=1)
    y = np.random.RandomState(2).randint(0, 5, size=(a.B, a.T)).astype(np.int32)
    P = a.B * a.T
    for H in (128, 256):
        sd = synth.synth_state_dict(0, num_features=F, gru_size=H)
        dt, stages, loss = ours(sd, x, y, H, a.steps, a.warmup)
        rows = [{"impl": "medaka_b200", "gru_size": H, "ms_per_step": dt * 1e3, "positions_per_s": P / dt,
                 "stage_ms": stages, "loss": loss}]
        if H == 128:
            dt8, st8, _ = ours(sd, x, y, H, max(1, a.steps // 2), 1, nb=8)
            rows.append({"impl": "medaka_b200 bptt 8 windows/CTA", "gru_size": H, "ms_per_step": dt8 * 1e3,
                         "positions_per_s": P / dt8, "stage_ms": st8})
        for tf32 in (True, False):
            dt, loss = torch_step(sd, x, y, H, a.steps, a.warmup, tf32)
            rows.append({"impl": "torch cudnn tf32=%s" % tf32, "gru_size": H, "ms_per_step": dt * 1e3,
                         "positions_per_s": P / dt, "loss": loss})
        for r in rows:
            r.update(B=a.B, T=a.T, F=F, card=gpu)
            print(json.dumps(r), flush=True)
        results += rows
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
