"""Variant annotation (medaka_b200.annotate): the CPU restatement against the reference's literals, and the GPU path
against both, on the reference's amplicon fixture and on synthetic data built to hit every trimming and tie rule."""
import importlib.util
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest

from medaka_b200 import annotate as mann
from medaka_b200.variant import Variant
from tests import annotate_oracle as ao
from tests import bamutil

HERE = os.path.dirname(os.path.abspath(__file__))
MAKER = os.path.join(HERE, "golden", "make_annotate_golden.py")
spec = importlib.util.spec_from_file_location("make_annotate_golden", MAKER)
golden = importlib.util.module_from_spec(spec)
spec.loader.exec_module(golden)


def _fixture():
    from medaka_b200 import stitch
    variants = golden.read_vcf(os.path.join(golden.DATA, "test_annotate.vcf"))
    ref = stitch.read_fasta(os.path.join(golden.DATA, "test_annotate_ref.fasta"))
    return variants, ref, os.path.join(golden.DATA, "test_annotate.bam")


def test_golden_maker_runs_clean():
    r = subprocess.run([sys.executable, MAKER], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "annotate golden OK" in r.stdout


def test_oracle_reproduces_reference_annotation():
    variants, ref, bam = _fixture()
    _, records = ao.read_bam(bam)
    got = ao.annotate(variants, ref, records, read_group=golden.READ_GROUP, pad=golden.PAD, dpsp=True)
    assert got == golden.expected_info()
    assert [v.chrom for v in variants] == ["MN908947.3"] * 3 + ["Duplicate"] * 3


def test_padded_haplotypes_and_alignment_literals():
    for (pos, r, a), pad, pref, palt, start, end in golden.PADDED_CASES:
        haps, region = ao.get_padded_haplotypes(Variant("c", pos, r, alt=a), golden.PADDED_REF, pad)
        assert (haps[0], haps[1], region) == (pref, palt, (start, end))
    with pytest.raises(ValueError):
        ao.get_padded_haplotypes(Variant("c", 2, "GT", alt="G"), golden.PADDED_REF, 2)
    haps = [golden.strip(h) for h, _ in golden.ALIGN_HAPS]
    assert ao.align_read_to_haps(golden.ALIGN_READ, haps) == [s for _, s in golden.ALIGN_HAPS]


def test_score_table():
    t = mann.SCORE_TABLE
    assert t.shape == (16, 16) and np.array_equal(t, t.T)
    acgt = [mann.NT16.index(c) for c in "ACGT"]
    block = t[np.ix_(acgt, acgt)]
    assert (np.diag(block) == 5).all() and (block[~np.eye(4, dtype=bool)] == -4).all()
    assert np.array_equal(t[0], t[15]) and t[15, 15] == -1      # '=' scores as N
    assert mann.nt16_code("x") == 15 and mann.nt16_code("u") == 15 and mann.nt16_code("g") == 4
    meta = mann.annotation_meta(pad=25)
    assert [m[1] for m in meta] == ["DP", "DPS", "DPSP", "SR", "AR", "SC"]
    assert "+-25" in meta[2][4] and "match 5, mismatch -4, open 5, extend 3" in meta[5][4]


def _gotoh(read, hap, go=5, ge=3):
    """Plain three-matrix Gotoh local alignment, one cell at a time."""
    t = mann.SCORE_TABLE
    m, n = len(read), len(hap)
    neg = -(1 << 28)
    H = [[0] * (n + 1) for _ in range(m + 1)]
    E = [[neg] * (n + 1) for _ in range(m + 1)]
    F = [[neg] * (n + 1) for _ in range(m + 1)]
    best = 0
    for i in range(1, m + 1):
        for j in range(1, n + 1):
            E[i][j] = max(E[i][j - 1] - ge, H[i][j - 1] - go)
            F[i][j] = max(F[i - 1][j] - ge, H[i - 1][j] - go)
            s = t[mann.nt16_code(read[i - 1]), mann.nt16_code(hap[j - 1])]
            H[i][j] = max(0, H[i - 1][j - 1] + int(s), E[i][j], F[i][j])
            best = max(best, H[i][j])
    return best


def test_batched_scores_equal_cell_by_cell_gotoh():
    rng = random.Random(3)
    alphabet = "ACGT" * 6 + "NRYKM=SWBDHV"
    pairs = []
    for _ in range(300):
        hap = "".join(rng.choice(alphabet) for _ in range(rng.randint(1, 45)))
        read = list(hap[rng.randint(0, len(hap) // 3):])
        for _ in range(rng.randint(0, 6)):
            k = rng.randrange(len(read) + 1)
            op = rng.random()
            if op < 0.4 and read:
                read[min(k, len(read) - 1)] = rng.choice(alphabet)
            elif op < 0.7:
                read[k:k] = [rng.choice("ACGT") for _ in range(rng.randint(1, 6))]
            else:
                del read[k:k + rng.randint(1, 6)]
        pairs.append(("".join(read) or "A", hap))
    got = ao.sw_scores(pairs, cells_per_batch=2000)
    assert got.tolist() == [_gotoh(r, h) for r, h in pairs]


def test_ref_mismatch_raises(tmp_path):
    path = str(tmp_path / "x.bam")
    bamutil.write_bam(path, [("c", 100)], [dict(ref=0, pos=0, cigar="50M", seq="A" * 50)])
    with pytest.raises(ValueError):
        mann.annotate([Variant("c", 10, "C", alt="A")], {"c": "A" * 100}, path)


# ---------------------------------------------------------------------------------------------------------------------
# synthetic data

BASES = "ACGT"
PAD = 25


def _read_from(rng, contig, start, end, haplotype_edit=None):
    """A read over contig[start, end) with random M/I/D runs, clips and base errors; haplotype_edit = (pos, ref_len,
    alt) makes it carry that allele.  Returns (pos, cigar string, seq)."""
    ops, seq = [], []
    if rng.random() < 0.3:
        n = rng.randint(1, 20)
        ops.append((n, "S"))
        seq += [rng.choice(BASES) for _ in range(n)]
    if rng.random() < 0.2:
        ops.insert(0, (rng.randint(1, 30), "H"))
    x = start
    while x < end:
        if haplotype_edit and x == haplotype_edit[0]:
            p, rl, alt = haplotype_edit
            # the allele as a match of the shared first base plus an insertion or deletion of the rest
            k = min(rl, len(alt))
            for i in range(k):
                seq.append(alt[i] if rng.random() > 0.03 else rng.choice(BASES))
                ops.append((1, "M"))
            if len(alt) > rl:
                seq += list(alt[k:])
                ops.append((len(alt) - rl, "I"))
            elif rl > len(alt):
                ops.append((rl - len(alt), "D"))
            x = p + rl
            continue
        r = rng.random()
        if r < 0.02:
            n = rng.randint(1, 4)
            ops.append((n, "I"))
            seq += [rng.choice(BASES) for _ in range(n)]
        elif r < 0.04 and x > start:
            n = min(rng.randint(1, 4), end - x)
            ops.append((n, "D"))
            x += n
        else:
            n = min(rng.randint(1, 12), end - x)
            if haplotype_edit and x < haplotype_edit[0] < x + n:
                n = haplotype_edit[0] - x
            for i in range(n):
                c = contig[x + i]
                seq.append(c if rng.random() > 0.03 else rng.choice("ACGTNRYKM"))
            ops.append((n, rng.choice("MMMM=X")))
            x += n
    if ops and ops[-1][1] == "D":
        ops.append((1, "M"))
        seq.append(contig[x] if x < len(contig) else "A")
    if rng.random() < 0.3:
        n = rng.randint(1, 20)
        ops.append((n, "S"))
        seq += [rng.choice(BASES) for _ in range(n)]
    if rng.random() < 0.2:
        ops.append((rng.randint(1, 30), "H"))
    merged = []
    for n, op in ops:
        if merged and merged[-1][1] == op:
            merged[-1] = (merged[-1][0] + n, op)
        else:
            merged.append((n, op))
    return start, "".join("%d%s" % (n, op) for n, op in merged), "".join(seq)


def _synthetic(seed, n_var=1500, length=120000, depth=12):
    rng = random.Random(seed)
    contig = "".join(rng.choice(BASES) for _ in range(length))
    contig = "".join(c if rng.random() > 0.002 else rng.choice("NRYSW") for c in contig)    # N and IUPAC in the draft
    positions = sorted(rng.sample(range(1, length - 60), n_var - 6))
    positions += [0, 3, length - 1, length - 2, length - 30]          # within pad of either contig end
    variants = []
    for p in sorted(set(positions)):
        r = rng.random()
        if r < 0.5:
            rl, alts = 1, [rng.choice([b for b in BASES if b != contig[p]])]
        elif r < 0.7:
            rl = 1
            alts = [contig[p] + "".join(rng.choice(BASES) for _ in range(rng.randint(1, 50)))]
        elif r < 0.9:
            rl = min(rng.randint(2, 51), length - p)
            alts = [contig[p]]
        elif r < 0.95:
            rl, alts = 1, [rng.choice(BASES), rng.choice(BASES) + "A"]                         # 2-alt records
        else:
            rl = 1
            alts = [contig[p], contig[p]] if r < 0.97 else [rng.choice(BASES)] * 2            # ties over 2 or 3 haps
        variants.append(Variant("ctg", p, contig[p:p + rl], alt=alts))
    # one deletion whose REF haplotype is longer than 2 kb, away from the others
    big = length // 2
    variants = [v for v in variants if not (big - 60 <= v.pos <= big + 2200)]
    variants.append(Variant("ctg", big, contig[big:big + 2100], alt=[contig[big]]))
    variants.sort(key=lambda v: v.pos)

    records = []
    rgs = ["A"] * 8 + ["B", None]
    n_reads = depth * length // 700
    for _ in range(n_reads):
        s = rng.randrange(0, length - 50)
        e = min(length, s + rng.randint(60, 1400))
        v = variants[rng.randrange(len(variants))]
        edit = None
        if rng.random() < 0.5 and s < v.pos and v.pos + len(v.ref) < e and v.ref != v.alt[0]:
            edit = (v.pos, len(v.ref), v.alt[0])
        records.append((s, e, edit))
    for _ in range(6):                                              # reads over the long deletion
        s = big - rng.randint(30, 200)
        records.append((s, min(length, big + 2100 + rng.randint(30, 200)), (big, 2100, contig[big]) if _ % 2 else None))
    out = []
    for s, e, edit in records:
        pos, cig, seq = _read_from(rng, contig, s, e, edit)
        tags = {}
        rg = rng.choice(rgs)
        if rg:
            tags["RG"] = rg
        flag = 16 if rng.random() < 0.5 else 0
        if rng.random() < 0.03:
            flag |= rng.choice([0x4, 0x100, 0x400, 0x800, 0x200])
        out.append(dict(ref=0, pos=pos, cigar=cig, seq=seq, flag=flag, mapq=0 if rng.random() < 0.03 else 60, tags=tags,
                        query_name="r%d" % len(out)))
    out += _edge_reads(contig, variants)
    out.sort(key=lambda r: r["pos"])
    for r in out:
        assert len(r["seq"]) == sum(int(n) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", r["cigar"]) if op in "MIS=X")
    return contig, variants, out


def _edge_reads(contig, variants):
    """Reads placed on the window edges of the first SNVs with room around them."""
    out = []
    snvs = [v for v in variants if len(v.ref) == 1 and 200 < v.pos < len(contig) - 200][:40:4]

    def rec(pos, cig, seq, flag=0):
        return dict(ref=0, pos=pos, cigar=cig, seq=seq, flag=flag, mapq=60, tags={"RG": "A"},
                    query_name="edge%d" % len(out))
    for v in snvs:
        rs, re_ = v.pos - PAD, v.pos + 1 + PAD
        s = rs - 40
        full = contig[s:re_ + 40]
        # ends exactly at rend (rejected), and one base further (kept)
        out.append(rec(s, "%dM" % (re_ - s), contig[s:re_]))
        out.append(rec(s, "%dM" % (re_ + 1 - s), contig[s:re_ + 1], flag=16))
        # starts exactly at rstart, and one base later (rejected)
        out.append(rec(rs, "%dM" % (re_ + 10 - rs), contig[rs:re_ + 10]))
        out.append(rec(rs + 1, "%dM" % (re_ + 10 - rs - 1), contig[rs + 1:re_ + 10]))
        # rstart and rend inside deletions, and inside insertions
        a, b = rs - s - 2, re_ - s - 2
        out.append(rec(s, "%dM5D%dM5D%dM" % (a, b - a - 5, len(full) - b - 5), full[:a] + full[a + 5:b] + full[b + 5:]))
        out.append(rec(s, "5S%dM3I%dM4I%dM7H" % (rs - s, re_ - rs, len(full) - (re_ - s)),
                       "ACGTA" + full[:rs - s] + "GGG" + full[rs - s:re_ - s] + "TTTT" + full[re_ - s:]))
        # a deletion over the whole window: trimmed length 0 or 1 (both dropped), or 2 (kept)
        out.append(rec(rs - 5, "5M%dD10M" % (re_ + 1 - rs), contig[rs - 5:rs] + contig[re_ + 1:re_ + 11]))
        out.append(rec(rs - 5, "5M%dD10M" % (re_ - rs), contig[rs - 5:rs] + contig[re_:re_ + 10]))
        out.append(rec(rs - 5, "5M%dD10M" % (re_ - 1 - rs), contig[rs - 5:rs] + contig[re_ - 1:re_ + 9]))
        # a reference skip (rejected) and a padding operation (rejected)
        out.append(rec(s, "%dM2N%dM" % (10, len(full) - 10), full[:10] + full[12:] + "AA"))
        out.append(rec(s, "10M1P%dM" % (len(full) - 10), full))
    return out


def _write(tmp_path, contig, records):
    path = str(tmp_path / "synth.bam")
    bamutil.write_bam(path, [("ctg", len(contig))], records, member_size=60000)
    return path


def _oracle_records(records):
    return [dict(r, ref="ctg") for r in records]


@pytest.fixture(scope="module")
def synth(tmp_path_factory):
    contig, variants, records = _synthetic(seed=11)
    path = _write(tmp_path_factory.mktemp("ann"), contig, records)
    want = ao.annotate(variants, {"ctg": contig}, _oracle_records(records), read_group="A", pad=PAD, dpsp=True)
    return contig, variants, path, want


@pytest.mark.gpu
def test_gpu_reference_fixture():
    variants, ref, bam = _fixture()
    got = mann.annotate(variants, ref, bam, read_group=golden.READ_GROUP, pad=golden.PAD, dpsp=True)
    assert [v.info for v in got] == golden.expected_info()
    assert [(v.chrom, v.pos, v.ref, v.alt, v.qual, v.genotype_data) for v in got] == \
        [(v.chrom, v.pos, v.ref, v.alt, v.qual, v.genotype_data) for v in variants]
    shallow = mann.annotate(variants, ref, bam, read_group=golden.READ_GROUP, pad=golden.PAD)
    assert [v.info for v in shallow] == [{k: e[k] for k in ("DP", "DPS")} for e in golden.expected_info()]


@pytest.mark.gpu
def test_gpu_synthetic_parity(synth):
    contig, variants, path, want = synth
    got = mann.annotate(variants, {"ctg": contig}, path, read_group="A", pad=PAD, dpsp=True)
    bad = [(v, g.info, w) for v, g, w in zip(variants, got, want) if g.info != w]
    assert not bad, (len(bad), bad[:3])
    # the data reach every rule: ties, spanning reads on both strands, uncovered variants
    assert sum(int(w["AR"].split(",")[0]) + int(w["AR"].split(",")[1]) for w in want) > 0
    assert any(int(w["DPSP"]) > 0 and len(w["SR"].split(",")) == 6 for w in want)
    long_hap = [w for v, w in zip(variants, want) if len(v.ref) > 2000]
    assert long_hap and int(long_hap[0]["DPSP"]) > 0


@pytest.mark.gpu
def test_gpu_chunking_and_repeats(synth):
    contig, variants, path, want = synth
    shuffled = list(variants)
    random.Random(5).shuffle(shuffled)
    for chunk_size in (997, 20000, 500000):
        got = mann.annotate(shuffled, {"ctg": contig}, path, read_group="A", pad=PAD, dpsp=True,
                            chunk_size=chunk_size)
        assert [g.info for g in got] == [want[variants.index(v)] for v in shuffled]
    from medaka_b200 import bam as mbam
    with mbam.BamFile(path) as fh:
        runs = [[g.info for g in mann.annotate(variants, {"ctg": contig}, fh, read_group="A", pad=PAD, dpsp=True)]
                for _ in range(2)]
    assert runs[0] == runs[1] == want
    depth_only = mann.annotate(variants, {"ctg": contig}, path, read_group="A", pad=PAD, dpsp=False)
    assert [g.info for g in depth_only] == [{k: w[k] for k in ("DP", "DPS")} for w in want]


@pytest.mark.gpu
def test_gpu_no_read_group_and_other_pad(synth):
    contig, variants, path, _ = synth
    vs = variants[::7]
    _, _, records = _synthetic(seed=11)
    want = ao.annotate(vs, {"ctg": contig}, _oracle_records(records), read_group=None, pad=7, dpsp=True)
    got = mann.annotate(vs, {"ctg": contig}, path, read_group=None, pad=7, dpsp=True)
    assert [g.info for g in got] == want
