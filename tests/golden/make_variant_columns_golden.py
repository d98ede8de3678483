"""Record the reference's own variant_columns (src/medaka_rnn_variants.c:28-55) on 20 seeded random cases.

Run:  make -C oracle REF=<medaka source checkout>  &&  python tests/golden/make_variant_columns_golden.py
      (or build with MEDAKA_REFERENCE=<medaka source checkout> python __graft_entry__.py)
Writes tests/golden/variant_columns.npz: the concatenated inputs (minor offsets, reference and predicted labels),
the C function's boolean output, and the length of every case.
"""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    lib = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libmedaka_rnn_variants.so"))
    lib.variant_columns.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_size_t]
    lib.variant_columns.restype = None
    rs = np.random.RandomState(9)
    minors, refs, preds, outs, lens = [], [], [], [], []
    for _ in range(20):
        n = int(rs.randint(1, 3000))
        is_minor = rs.uniform(size=n) < 0.3
        is_minor[0] = False
        idx = np.arange(n)
        last_major = np.maximum.accumulate(np.where(~is_minor, idx, -1))
        minor = np.ascontiguousarray(idx - last_major, dtype=np.uintp)
        ref = rs.randint(0, 5, n)
        pred = np.where(rs.uniform(size=n) < 0.85, ref, rs.randint(0, 5, n))
        r32, p32 = np.ascontiguousarray(ref, dtype=np.int32), np.ascontiguousarray(pred, dtype=np.int32)   # wchar_t
        out = np.zeros(n, dtype=np.bool_)
        lib.variant_columns(minor.ctypes.data, r32.ctypes.data, p32.ctypes.data, out.ctypes.data, n)
        minors.append(minor.astype(np.int32))
        refs.append(ref.astype(np.int8))
        preds.append(pred.astype(np.int8))
        outs.append(out)
        lens.append(n)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "variant_columns.npz"), lengths=np.array(lens, np.int64),
                        minor=np.concatenate(minors), ref=np.concatenate(refs), pred=np.concatenate(preds),
                        out=np.concatenate(outs))


if __name__ == "__main__":
    main()
