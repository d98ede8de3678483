"""Golden vectors of the reference's training loop: the REAL reference GRUModel (``medaka.models.model_from_dict``,
normalise = False as run_epoch sets it for CrossEntropyLoss) through three steps of

    model.process_batch(batch, CrossEntropyLoss())  ->  loss.backward()  ->  ClipGrad()(parameters)
    ->  RMSprop(lr 0.001, alpha 0.9, eps 1e-7, momentum 0)  ->  linear_warmup_cosine_decay()(...).step()

(medaka/training.py run_training's defaults, medaka/torch_ext.py run_epoch's order) at gru_size 128 and 256, on the CPU
in fp32.  The schedule is sized for one epoch of STEPS_PER_EPOCH batches, so its default 500-step warmup is in force.

Run:  python tests/golden/make_train_golden.py     (needs the reference checkout; writes tests/golden/train_steps.npz)

The reference is imported unmodified behind the stand-ins of make_golden.py.  Only seeds, shapes and outputs are
stored: the weights regenerate from oracle.synth.synth_state_dict(SEED, num_features=F, gru_size=H), the batch of step s
from oracle.synth.synth_features(B, T, F, seed=10 + s) and labels RandomState(20 + s).randint(0, 5, (B, T)).  Per step:
loss, pre-clip gradient norm, clip threshold (2 x the median of ClipGrad's buffer) and learning rate; float64 sum and
sum of squares of every gradient tensor at step 1 (before clipping) and of every weight tensor after step 3, and of
every weight tensor's change over the three steps.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SEED, F, B, T, STEPS, STEPS_PER_EPOCH = 4, 10, 3, 80, 3, 1000


def batch_arrays(step):
    import numpy as np
    from oracle import synth
    x = synth.synth_features(B, T, F, seed=10 + step)
    y = np.random.RandomState(20 + step).randint(0, 5, size=(B, T))
    return x, y


def main():
    from make_golden import install_stubs
    install_stubs()
    import numpy as np
    import torch
    import medaka.models as ref_models
    import medaka.torch_ext as ref_ext
    from oracle import synth

    torch.set_num_threads(8)
    meta = "medaka v%s, torch %s, numpy %s" % (__import__('medaka').__version__, torch.__version__, np.__version__)
    print(meta)
    out = {}
    for H in (128, 256):
        model = ref_models.model_from_dict({"type": "GRUModel", "kwargs": {"num_features": F, "num_classes": 5,
                                                                           "gru_size": H}})
        sd = synth.synth_state_dict(SEED, num_features=F, gru_size=H)
        model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        model.train()
        model.normalise = False                      # torch_ext.run_epoch with CrossEntropyLoss
        keys = list(model.state_dict().keys())
        w0 = {k: v.detach().double().clone() for k, v in model.state_dict().items()}
        loss_fn = torch.nn.CrossEntropyLoss()
        optimizer = torch.optim.RMSprop(model.parameters(), lr=0.001, alpha=0.9, eps=1e-07, momentum=0.0)
        clip = ref_ext.ClipGrad()
        sched = ref_ext.linear_warmup_cosine_decay()(optimizer, [None] * STEPS_PER_EPOCH, 1, 0)
        steps = []
        for s in range(STEPS):
            x, y = batch_arrays(s)
            batch = ref_ext.Batch(counts_matrix=torch.from_numpy(x), labels=torch.from_numpy(y))
            optimizer.zero_grad()
            loss, metrics = model.process_batch(batch, loss_fn)
            loss.backward()
            if s == 0:
                named = dict(model.named_parameters())
                g = [named[k].grad.detach().double() for k in keys]
                out["h%d_grad_sum" % H] = np.array([float(v.sum()) for v in g])
                out["h%d_grad_sumsq" % H] = np.array([float((v * v).sum()) for v in g])
            threshold = clip.factor * np.quantile(clip.buffer, clip.quantile)
            lr = sched.get_last_lr()[0]
            norm = clip(model.parameters())
            optimizer.step()
            sched.step()
            steps.append([loss.item(), norm, threshold, lr, metrics["n_model_correct"]])
            print("H=%d step %d: loss %.6f norm %.6f threshold %g lr %g" % (H, s, loss.item(), norm, threshold, lr))
        w3 = {k: v.detach().double() for k, v in model.state_dict().items()}
        out["h%d_steps" % H] = np.array(steps)
        out["h%d_weight_sum" % H] = np.array([float(w3[k].sum()) for k in keys])
        out["h%d_weight_sumsq" % H] = np.array([float((w3[k] ** 2).sum()) for k in keys])
        out["h%d_delta_sum" % H] = np.array([float((w3[k] - w0[k]).sum()) for k in keys])
        out["h%d_delta_sumsq" % H] = np.array([float(((w3[k] - w0[k]) ** 2).sum()) for k in keys])
        out["keys"] = np.array(keys)
    out["args"] = np.array([SEED, F, B, T, STEPS, STEPS_PER_EPOCH])
    np.savez_compressed(os.path.join(HERE, "train_steps.npz"), meta=meta, **out)


if __name__ == "__main__":
    main()
