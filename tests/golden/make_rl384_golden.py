"""Golden outputs of the REFERENCE's read-level network at lstm_size = 384 (build container only).

Run:  python tests/golden/make_rl384_golden.py     (needs /root/reference; writes tests/golden/rl_forward_lstm384.npz)

Every read-level model medaka ships is named ``..._rl_lstm384_{dwells,no_dwells}``.  The archives themselves are Git-LFS
stubs in the reference checkout, so their constructor arguments cannot be read: the cases below take lstm_size = 384 from
the name and the class defaults for everything else (cnn_size = 128, kernel_sizes = [1, 17], mean pooling,
bidirectional).  As in make_rl_golden.py the reference's LatentSpaceLSTM is imported unmodified, loaded with seeded
parameters (oracle/rl_oracle.py::synth_rl_state_dict) and run in eval mode; the restatement in oracle/rl_oracle.py is
asserted against it.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden  # noqa: E402
from oracle import rl_oracle  # noqa: E402

LSTM_SIZE = 384
CASES = {            # name: (seed, B, P, D, use_dwells, gain)
    "small": (10, 2, 96, 7, False, 1.0),
    "deep": (11, 1, 300, 40, False, 1.0),
    "dwells": (12, 3, 130, 9, True, 1.0),
    "hot": (13, 2, 500, 12, False, 2.5),
    "long": (14, 1, 2100, 6, False, 1.0),
}


def build_oracle(sd, use_dwells):
    """The restatement at lstm_size = 384 (what rl_oracle.build makes of a 384 state dict)."""
    m = rl_oracle.LatentSpaceLSTM(lstm_size=LSTM_SIZE, use_dwells=use_dwells)
    m.load_state_dict(sd)
    m.eval()
    return m


def case_inputs(seed, B, P, D, dw, gain):
    sd = rl_oracle.synth_rl_state_dict(seed, lstm_size=LSTM_SIZE, use_dwells=dw, gain=gain)
    x = rl_oracle.synth_rl_features(B, P, D, use_dwells=dw, seed=100 + seed)
    return sd, x


def main():
    make_golden.install_stubs()
    sys.path.insert(0, "/root/reference")
    from medaka.architectures.latent_space_lstm import LatentSpaceLSTM
    out = {}
    for name, (seed, B, P, D, dw, gain) in CASES.items():
        sd, x = case_inputs(seed, B, P, D, dw, gain)
        ref = LatentSpaceLSTM(lstm_size=LSTM_SIZE, use_dwells=dw)
        ref.load_state_dict(sd)
        ref.eval()
        torch.set_num_threads(8)
        with torch.inference_mode():
            probs = ref(torch.from_numpy(x)).numpy()
        mine = rl_oracle.predict(build_oracle(sd, dw), x)
        err = float(np.abs(mine - probs).max())
        assert err < 2e-6, (name, err)
        out[name + "_args"] = np.array([seed, B, P, D, int(dw), gain], dtype=np.float64)
        out[name + "_probs"] = probs
        print(name, probs.shape, "restatement vs reference %.2e" % err, "mean max prob %.3f" % probs.max(-1).mean())
    np.savez_compressed(os.path.join(HERE, "rl_forward_lstm384.npz"), **out)


if __name__ == "__main__":
    main()
