"""The GRU engine's weight packer (medaka_b200/csrc/gru_pack.cuh), run on the CPU by a native driver
(tests/native/gru_pack_check.cu): every array the kernels read, checked bit for bit at the indices they read it."""
import os
import subprocess

import numpy as np
import pytest

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 128
SCALE = np.array([-1.4426950408889634, -1.4426950408889634, 2.8853900817779268], np.float32)   # gate_scale(r, z, n)
F32 = ["w_in_packed", "bias_gi", "b_hn", "bias_gi_tc", "b_hn_tc", "w_hh_t"]
F16 = ["w_hh_tm", "w_x_tm", "w_in_tc"]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    import __graft_entry__
    exe = str(tmp_path_factory.mktemp("gru_pack") / "gru_pack_check")
    subprocess.run([__graft_entry__._nvcc(), "-std=c++17", "-O1", "-o", exe,
                    os.path.join(ROOT, "tests", "native", "gru_pack_check.cu")], check=True, capture_output=True)
    return exe


def _pack(exe, sd, F, tmp_path):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for layer in range(2):
            for sfx in ("", "_reverse"):
                for name in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    f.write(np.ascontiguousarray(sd["gru.%s_l%d%s" % (name, layer, sfx)], np.float32).tobytes())
    r = subprocess.run([exe, str(F), src, dst], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw, off, layers = open(dst, "rb").read(), 0, []
    for _ in range(2):
        arrays = {}
        for name in F32 + F16:
            n = int(np.frombuffer(raw, np.int64, 1, off)[0])
            dt = np.float32 if name in F32 else np.float16
            arrays[name] = np.frombuffer(raw, dt, n, off + 8)
            off += 8 + n * np.dtype(dt).itemsize
        layers.append(arrays)
    assert off == len(raw)
    return layers


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _hi_lo(x):
    """fp16 hi / lo planes of float32 x: hi = fp16(x), lo = fp16(x - hi)."""
    hi = x.astype(np.float16)
    return np.stack([hi, (x - hi.astype(np.float32)).astype(np.float16)])


@pytest.mark.parametrize("F", [10, 20])
def test_gru_pack_layouts(driver, tmp_path, F):
    sd = synth.synth_state_dict(3, num_features=F)
    layers = _pack(driver, sd, F, tmp_path)
    for layer, got in enumerate(layers):
        nin = F if layer == 0 else 2 * H
        w_ih = [sd["gru.weight_ih_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        w_hh = [sd["gru.weight_hh_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        b_ih = [sd["gru.bias_ih_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        b_hh = [sd["gru.bias_hh_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        # input weights: the row stack of both directions, [768][in]
        assert np.array_equal(_bits(got["w_in_packed"].reshape(6 * H, nin)), _bits(np.concatenate(w_ih)))
        # biases: r and z get b_ih + b_hh, n gets b_ih; b_hn is the n part of b_hh; the _tc copies times gate_scale
        bias = np.concatenate([np.concatenate([bi[:2 * H] + bh[:2 * H], bi[2 * H:]]) for bi, bh in zip(b_ih, b_hh)])
        b_hn = np.stack([bh[2 * H:] for bh in b_hh])
        assert np.array_equal(_bits(got["bias_gi"]), _bits(bias))
        assert np.array_equal(_bits(got["b_hn"].reshape(2, H)), _bits(b_hn))
        assert np.array_equal(_bits(got["bias_gi_tc"].reshape(2, 3, H)), _bits(bias.reshape(2, 3, H) * SCALE[:, None]))
        assert np.array_equal(_bits(got["b_hn_tc"].reshape(2, H)), _bits(b_hn * SCALE[2]))
        # recurrent weights: W_hh^T [d][k][384] for the fp32 path, fp16 hi / lo of W_hh * gate_scale [d][part][gate][j][k]
        assert np.array_equal(_bits(got["w_hh_t"].reshape(2, H, 3 * H)), _bits(np.stack([w.T for w in w_hh])))
        w_hh_tm = np.stack([_hi_lo(w.reshape(3, H, H) * SCALE[:, None, None]) for w in w_hh])
        assert np.array_equal(_bits(got["w_hh_tm"].reshape(2, 2, 3, H, H)), _bits(w_hh_tm))
        # layer 0 at F <= 16: W_ih as [d][part][gate][j][16], zero beyond F; absent otherwise
        if layer == 0 and F <= 16:
            pad = [np.pad(w, ((0, 0), (0, 16 - F))).reshape(3, H, 16) * SCALE[:, None, None] for w in w_ih]
            w_x_tm = got["w_x_tm"].reshape(2, 2, 3, H, 16)
            assert np.array_equal(_bits(w_x_tm), _bits(np.stack([_hi_lo(x) for x in pad])))
            assert not w_x_tm[..., F:].astype(np.float32).any()
        else:
            assert got["w_x_tm"].size == 0
        # layer 1: W_ih as [blk = dir * 3 + gate][part][j][k 256]
        if layer == 1:
            w_in_tc = np.stack([_hi_lo(w.reshape(3, H, nin)[g] * SCALE[g]) for w in w_ih for g in range(3)])
            assert np.array_equal(_bits(got["w_in_tc"].reshape(6, 2, H, nin)), _bits(w_in_tc))
        else:
            assert got["w_in_tc"].size == 0
