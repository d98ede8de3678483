"""Golden vectors of the reference's training loop for the read-level model: the REAL reference LatentSpaceLSTM
(``medaka.models.model_from_dict``, model.train(), normalise = False as run_epoch sets it) through three steps of

    model.process_batch(batch, CrossEntropyLoss())  ->  loss.backward()  ->  ClipGrad()(parameters)
    ->  RMSprop(lr 0.001, alpha 0.9, eps 1e-7, momentum 0)  ->  linear_warmup_cosine_decay()(...).step()

on the CPU in fp32, at lstm_size 128 and 384 and with dwells at 128.  The batches are int8 read_level_features given
to Batch directly: strands -1 and 1, ragged reads, an empty read in the middle of a window, padding reads, and
P = 37, a multiple of no tile.

Run:  python tests/golden/make_rl_train_golden.py     (needs the reference checkout; writes tests/golden/rl_train_steps.npz)

Only seeds, shapes and outputs are stored: the weights regenerate from oracle.rl_oracle.synth_rl_state_dict, the batch
of step s from rl_batch(case, s).  Per case: per-step loss, pre-clip norm, clip threshold, learning rate and
model-correct count; float64 sum and sum of squares of every gradient at step 1, of every weight and buffer after step
3, and of a fresh model_from_dict's state dict under torch.manual_seed(SEED).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SEED, STEPS, STEPS_PER_EPOCH, P = 5, 3, 1000, 37
# (name, lstm_size, use_dwells, B, D)
CASES = [("h128", 128, False, 3, 6), ("h384", 384, False, 2, 5), ("h128dw", 128, True, 3, 6)]


def rl_batch(case, step):
    """int8 [B, P, D, F] features and labels [B, P] of one step of a case"""
    import numpy as np
    from oracle import rl_oracle
    _, H, dw, B, D = case
    x = rl_oracle.synth_rl_features(B, P, D, use_dwells=dw, seed=30 + step, empty_rows=2)
    rs = np.random.RandomState(40 + step)
    on = x[..., 0] != 0
    x[..., 2] = np.where(on & (x[..., 2] == 0), -1, x[..., 2])      # strand -1 / 1 on real cells
    x[0, :, 1, :] = 0                                               # an empty read between real ones
    y = rs.randint(0, 5, size=(B, P))
    return x, y


def model_dict(case):
    _, H, dw, _, _ = case
    return {"type": "LatentSpaceLSTM", "kwargs": {"num_classes": 5, "lstm_size": H, "cnn_size": 128,
                                                  "use_dwells": dw}}


def main():
    from make_golden import install_stubs
    install_stubs()
    import numpy as np
    import torch
    import medaka.models as ref_models
    import medaka.torch_ext as ref_ext
    from oracle import rl_oracle

    torch.set_num_threads(8)
    meta = "medaka v%s, torch %s, numpy %s" % (__import__('medaka').__version__, torch.__version__, np.__version__)
    print(meta)
    out = {}
    for case in CASES:
        name, H, dw, B, D = case
        torch.manual_seed(SEED)
        fresh = ref_models.model_from_dict(model_dict(case))
        fsd = fresh.state_dict()
        out[name + "_keys"] = np.array(list(fsd.keys()))
        out[name + "_init_sum"] = np.array([float(v.double().sum()) for v in fsd.values()])
        out[name + "_init_sumsq"] = np.array([float((v.double() ** 2).sum()) for v in fsd.values()])
        model = ref_models.model_from_dict(model_dict(case))
        sd = rl_oracle.synth_rl_state_dict(SEED, lstm_size=H, use_dwells=dw)
        model.load_state_dict(sd)
        model.train()
        model.normalise = False
        keys = list(model.state_dict().keys())
        pkeys = [k for k, _ in model.named_parameters() if "read_level_conv.expansion_layer" not in k]
        loss_fn = torch.nn.CrossEntropyLoss()
        optimizer = torch.optim.RMSprop(model.parameters(), lr=0.001, alpha=0.9, eps=1e-07, momentum=0.0)
        clip = ref_ext.ClipGrad()
        sched = ref_ext.linear_warmup_cosine_decay()(optimizer, [None] * STEPS_PER_EPOCH, 1, 0)
        steps = []
        for s in range(STEPS):
            x, y = rl_batch(case, s)
            batch = ref_ext.Batch(read_level_features=torch.from_numpy(x), labels=torch.from_numpy(y))
            optimizer.zero_grad()
            loss, metrics = model.process_batch(batch, loss_fn)
            loss.backward()
            if s == 0:
                named = dict(model.named_parameters())
                assert named["read_level_conv.expansion_layer.weight"].grad is None
                g = [named[k].grad.detach().double() for k in pkeys]
                out[name + "_grad_keys"] = np.array(pkeys)
                out[name + "_grad_sum"] = np.array([float(v.sum()) for v in g])
                out[name + "_grad_sumsq"] = np.array([float((v * v).sum()) for v in g])
            threshold = clip.factor * np.quantile(clip.buffer, clip.quantile)
            lr = sched.get_last_lr()[0]
            norm = clip(model.parameters())
            optimizer.step()
            sched.step()
            steps.append([loss.item(), norm, threshold, lr, metrics["n_model_correct"]])
            print("%s step %d: loss %.6f norm %.6f threshold %g lr %g" % (name, s, loss.item(), norm, threshold, lr))
        w3 = {k: v.detach().double() for k, v in model.state_dict().items()}
        out[name + "_steps"] = np.array(steps)
        out[name + "_weight_sum"] = np.array([float(w3[k].sum()) for k in keys])
        out[name + "_weight_sumsq"] = np.array([float((w3[k] ** 2).sum()) for k in keys])
    out["args"] = np.array([SEED, STEPS, STEPS_PER_EPOCH, P])
    np.savez_compressed(os.path.join(HERE, "rl_train_steps.npz"), meta=meta, **out)


if __name__ == "__main__":
    main()
