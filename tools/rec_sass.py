#!/usr/bin/env python
"""Step-loop instruction mix of every rec_tc_kernel instantiation, from the compiled SASS.  Needs nvcc, no GPU.

    python tools/rec_sass.py [--json]

Compiles medaka_b200/csrc/gru_wg.cu with the build's flags (and -Xptxas -v) into a temporary directory, disassembles
it with cuobjdump -sass and, per instantiation rec_tc_kernel<NT, FUSE_X, OUT>, finds the step loop: the backward
branch that closes the loop holding the HGMMAs.  It counts per warp and step the instructions before the
WARPGROUP.DEPBAR that waits for the step's MMAs (issue side) and after it (gate math, h store, barrier), and by opcode:
HGMMA, MUFU (EX2 / RCP, after the wait), the shared-memory stores of the h tile (STS.U16, STSM) and the F2FP
conversions after the wait.  Registers and spill bytes come from ptxas.  Writes nothing outside the temporary directory.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OUT_NAMES = {0: "OUT_TILES", 1: "OUT_ROWS", 2: "OUT_LOGITS"}
LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?);")
KERNEL = re.compile(r"_ZN3mdk13rec_tc_kernelILi(\d)ELb(\d)ELi(\d)E")


def compile_and_dump(tmp):
    import __graft_entry__ as ge
    src = os.path.join(ge.CSRC, "gru_wg.cu")
    obj = os.path.join(tmp, "gru_wg.o")
    r = subprocess.run([ge._nvcc()] + ge.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit("nvcc failed:\n" + r.stdout + r.stderr)
    cuobjdump = os.path.join(os.path.dirname(ge._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def ptxas_resources(log):
    """{mangled name: (registers, spill store bytes, spill load bytes)} from the -Xptxas -v log."""
    res, cur, spill = {}, None, (0, 0)
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spill = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            res[cur] = (int(m.group(1)),) + spill
            cur, spill = None, (0, 0)
    return res


def split_functions(sass):
    funcs, name, body = {}, None, []
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            name, body = m.group(1), []
            continue
        m = LINE.search(line)
        if m and name:
            body.append((int(m.group(1), 16), m.group(2).strip()))
    if name:
        funcs[name] = body
    return funcs


def opcode(ins):
    ins = re.sub(r"^@!?U?P\w+\s+", "", ins)
    return ins.split()[0] if ins else ""


def step_loop(body):
    """(before, after): the instructions of the step loop up to and including its WARPGROUP.DEPBAR, and after it."""
    first_mma = next(a for a, i in body if opcode(i).startswith("HGMMA"))
    for idx, (addr, ins) in enumerate(body):
        m = re.match(r"(?:@!?U?P\w+\s+)?BRA\s+(?:`\(\.L_x_\d+\)\s*)?0x([0-9a-f]+)", ins)
        if not m:
            continue
        target = int(m.group(1), 16)
        if target <= first_mma < addr:
            loop = [(a, i) for a, i in body if target <= a <= addr]
            wait = [k for k, (a, i) in enumerate(loop) if opcode(i).startswith("WARPGROUP.DEPBAR")]
            if not wait:
                continue
            w = wait[-1]
            return loop[:w + 1], loop[w + 1:]
    raise RuntimeError("no step loop found")


def mix(before, after):
    ops_b = collections.Counter(opcode(i) for _, i in before)
    ops_a = collections.Counter(opcode(i) for _, i in after)
    both = ops_b + ops_a

    def count(ops, pred):
        return sum(n for o, n in ops.items() if pred(o))
    return {
        "before_wait": len(before), "after_wait": len(after),
        "HGMMA": count(both, lambda o: o.startswith("HGMMA")),
        "MUFU": count(ops_a, lambda o: o.startswith("MUFU")),
        "MUFU.EX2": count(ops_a, lambda o: o == "MUFU.EX2"),
        "MUFU.RCP": count(ops_a, lambda o: o == "MUFU.RCP"),
        "MUFU_before_wait": count(ops_b, lambda o: o.startswith("MUFU")),
        "STS.U16": count(ops_a, lambda o: o == "STS.U16"),
        "STSM": count(both, lambda o: o.startswith("STSM")),
        "F2FP": count(ops_a, lambda o: o.startswith("F2FP")),
        "FFMA+FMUL+FADD": count(ops_a, lambda o: o.split(".")[0] in ("FFMA", "FMUL", "FADD")),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", action="store_true", help="one JSON line instead of the table")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        log, sass = compile_and_dump(tmp)
    res = ptxas_resources(log)
    rows = []
    for name, body in split_functions(sass).items():
        m = KERNEL.match(name)
        if not m:
            continue
        nt, fx, out = int(m.group(1)), bool(int(m.group(2))), int(m.group(3))
        regs, sst, sld = res.get(name, (None, None, None))
        row = {"kernel": "rec_tc_kernel<%d,%s,%s>" % (nt, "true" if fx else "false", OUT_NAMES[out]),
               "registers": regs, "spill_store_bytes": sst, "spill_load_bytes": sld}
        row.update(mix(*step_loop(body)))
        rows.append(row)
    rows.sort(key=lambda r: r["kernel"])
    if args.json:
        print(json.dumps(rows))
        return
    cols = ["before_wait", "after_wait", "HGMMA", "MUFU", "MUFU.EX2", "MUFU.RCP", "STS.U16", "STSM", "F2FP",
            "FFMA+FMUL+FADD", "registers", "spill_store_bytes"]
    heads = ["before", "after", "HGMMA", "MUFU", "EX2", "RCP", "STS.U16", "STSM", "F2FP", "FP32", "regs", "spill"]
    w = max(len(r["kernel"]) for r in rows)
    print("per warp and step; MUFU, STS.U16, F2FP and FP32 (FFMA + FMUL + FADD) counted after the MMA wait")
    print("%-*s " % (w, "instantiation") + " ".join("%7s" % h for h in heads))
    for r in rows:
        print("%-*s " % (w, r["kernel"]) + " ".join("%7s" % r[c] for c in cols))


if __name__ == "__main__":
    main()
