"""Golden vectors of the default-trained model width: the REAL reference GRUModel at gru_size = 256, built by
``medaka.models.model_from_dict(DEFAULT_MODEL_DICT)`` (the model ``medaka train`` builds when no model is given) and run
through ``TorchModel.predict_on_batch``.

Run:  python tests/golden/make_gru256_golden.py     (needs the reference checkout; writes tests/golden/gru256_forward.npz)

The reference is imported unmodified behind the stand-ins of make_golden.py.  Only seeds, shapes and outputs are
stored: the weights regenerate from oracle.synth.synth_state_dict(seed, num_features=F, gru_size=256, head_gain,
rec_gain) and the features from oracle.synth.synth_features(B, T, F, seed=100 + seed).  The F = 20 case builds its
model from DEFAULT_MODEL_DICT with num_features replaced.
"""
import copy
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

# name, seed, B, T, F, head_gain, rec_gain
CASES = [
    ("default", 0, 3, 500, 10, 8.0, 1.0),
    ("f20", 1, 2, 300, 20, 8.0, 1.0),
    ("ragged", 2, 37, 41, 10, 8.0, 1.0),     # B not a multiple of the 16-window tile
    ("t1", 3, 19, 1, 10, 8.0, 1.0),          # one column
    ("short", 4, 17, 3, 10, 8.0, 1.0),
    ("hot", 5, 4, 400, 10, 24.0, 2.5),       # larger recurrent gain, sharper logits
]


def main():
    from make_golden import install_stubs
    install_stubs()
    import numpy as np
    import torch
    import medaka.models as ref_models
    from oracle import synth

    torch.set_num_threads(8)
    meta = "medaka v%s, torch %s, numpy %s, DEFAULT_MODEL_DICT %r" % (
        __import__('medaka').__version__, torch.__version__, np.__version__, ref_models.DEFAULT_MODEL_DICT)
    print(meta)
    assert ref_models.DEFAULT_MODEL_DICT["kwargs"]["gru_size"] == 256
    out = {}
    for name, seed, B, T, F, head_gain, rec_gain in CASES:
        d = copy.deepcopy(ref_models.DEFAULT_MODEL_DICT)
        d["kwargs"]["num_features"] = F
        model = ref_models.model_from_dict(d)
        sd = synth.synth_state_dict(seed, num_features=F, gru_size=256, head_gain=head_gain, rec_gain=rec_gain)
        model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        model.eval()
        feats = synth.synth_features(B, T, F, seed=100 + seed)

        class _Batch:
            counts_matrix = torch.from_numpy(feats)

        probs = model.predict_on_batch(_Batch())          # medaka/models.py:303-313
        model.normalise = False                            # gru.py:68-71 -> logits
        logits = model.predict_on_batch(_Batch())
        out[name + "_probs"] = probs.numpy()
        out[name + "_logits"] = logits.numpy()
        out[name + "_args"] = np.array([seed, B, T, F, head_gain, rec_gain], dtype=np.float64)
        print("forward", name, tuple(probs.shape), float(probs.max()))
    np.savez_compressed(os.path.join(HERE, "gru256_forward.npz"), meta=meta, **out)


if __name__ == "__main__":
    main()
