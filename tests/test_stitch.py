"""Consensus stitching (SURVEY.md section 8 f1): oracle and host planner against the reference's recorded results on
CPU; the device decode + compaction against both on the GPU (bytes must be identical)."""
import io
import json
import os

import numpy as np
import pytest

from medaka_b200 import stitch
from medaka_b200.common import OverlapException, Region, Sample
from oracle import labels_oracle, stitch_oracle, synth


def _golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "stitch.npz"))
    return {k: json.loads(str(g[k])) for k in g.files if k != "meta"}


def _samples(stream):
    return [Sample(ref_name=s['ref_name'], features=None, labels=None, ref_seq=None, positions=s['positions'],
                   label_probs=s['label_probs'], depth=s['depth']) for s in stream]


def _flatten(contigs):
    return [[[c[0][0], int(c[0][1]), int(c[0][2])], ''.join(c[1]), ''.join(c[2]), [len(x) for x in c[1]]]
            for c in contigs]


# The winning class's probability at the phred edges: 1, either side of the clip at 1 - 1e-7, and where -10 log10(1 - p)
# lands on an integer (the quality byte truncates it)
PHRED_EDGE_P = np.array([1.0, np.nextafter(np.float32(1 - 1e-7), np.float32(0)), np.float32(1 - 1e-7),
                         np.nextafter(np.float32(1 - 1e-7), np.float32(1)), 0.9, 0.99, 0.999, 0.9999, 0.99999],
                        np.float32)


def phred_edge_rows(cls=2):
    """5-class probability rows whose class cls (one per row, or one for all) takes the PHRED_EDGE_P values."""
    rows = np.repeat(((1 - PHRED_EDGE_P) / 4)[:, None], 5, axis=1).astype(np.float32)
    rows[np.arange(len(rows)), cls] = PHRED_EDGE_P
    return rows


def _cpu_decode(samples, pieces):
    """What decode_pieces must return, from the oracle's decode on the planned rows."""
    seqs, quals = [], []
    for p in pieces:
        s, q = labels_oracle.decode_consensus(samples[p.sample].label_probs[p.lo:p.hi], with_qualities=True)
        seqs.append(s)
        quals.append(q)
    return seqs, quals


def test_oracle_matches_reference(golden_dir):
    for name, rec in _golden(golden_dir).items():
        stream = synth.synth_stitch_stream(**rec["kwargs"])
        got = stitch_oracle.stitch_samples(stream, rec["start"], rec["end"], rec["min_depth"])
        assert _flatten(got) == rec["contigs"], name


def test_planner_matches_reference(golden_dir, monkeypatch):
    """The index-range plan + a CPU decode of the planned rows reproduces the reference contigs part by part."""
    monkeypatch.setattr(stitch, "decode_pieces", lambda samples, pieces, device=0, with_qualities=True:
                        _cpu_decode(samples, pieces))
    used_heuristic = 0
    for name, rec in _golden(golden_dir).items():
        samples = _samples(synth.synth_stitch_stream(**rec["kwargs"]))
        region = Region('contig1', rec["start"], rec["end"])
        got = stitch.stitch_samples(samples, None, region, rec["min_depth"])
        assert _flatten(got) == rec["contigs"], name
        joined = [[[c[0][0], int(c[0][1]), int(c[0][2])], ''.join(c[1]), ''.join(c[2])]
                  for c in stitch.collapse_neighbours(got)]
        assert joined == rec["collapsed"], name
        used_heuristic += sum(p.heuristic for p in stitch.plan_pieces(samples, rec["start"], rec["end"]))
    assert used_heuristic >= 3          # the ragged cases really went through the junction search


def test_junction_literals():
    """The reference's own overlap test vectors (medaka/test/test_sample.py:283-345)."""
    dt = [('major', int), ('minor', int)]
    pos1 = np.array([(0, 0), (0, 1), (1, 0), (2, 0), (2, 1), (2, 2), (3, 0), (4, 0), (4, 1), (4, 2), (4, 3),
                     (5, 0), (6, 0), (6, 1), (7, 0), (7, 1)], dtype=dt)
    others = [
        np.array([(3, 0), (4, 0), (4, 1), (4, 2), (4, 3), (5, 0), (6, 0), (7, 0), (7, 1), (8, 0)], dtype=dt),
        np.array([(3, 0), (4, 0), (4, 1), (4, 2), (5, 0), (5, 1), (6, 0), (6, 1), (7, 0), (7, 1), (8, 0), (9, 0),
                  (10, 0), (10, 1), (10, 2)], dtype=dt),
    ]
    # equal structure is cut at the mid-point of the overlap
    same = pos1[6:].copy()
    e1, s2, heur = stitch.junction(pos1, np.concatenate([same, np.array([(8, 0)], dtype=dt)]))
    assert not heur and e1 == 6 + 5 and s2 == 5
    for other in others:
        e1, s2, heur = stitch.junction(pos1, other)
        assert heur and tuple(pos1[e1]) == tuple(other[s2]) and pos1[e1]['minor'] == 0
    # too few major positions in the overlap to search for a junction
    with pytest.raises(OverlapException):
        stitch.junction(pos1, np.array([(6, 0), (7, 0), (7, 1), (7, 2), (8, 0)], dtype=dt))


def test_plan_errors_and_edges():
    stream = synth.synth_stitch_stream(seed=11)
    samples = _samples(stream)
    assert stitch.plan_pieces([]) == []
    with pytest.raises(OverlapException):                   # out-of-order stream
        stitch.plan_pieces(samples[::-1])
    other = samples[1].amend(ref_name='contig2')
    with pytest.raises(OverlapException):
        stitch.plan_pieces([samples[0], other])
    # region outside the data -> nothing
    assert stitch.plan_pieces(samples, start=10 ** 7, end=10 ** 7 + 5) == []
    assert stitch.plan_pieces(samples, start=0, end=10) == []
    # pieces tile the region: consecutive pieces abut exactly
    pieces = stitch.plan_pieces(samples)
    for a, b in zip(pieces[:-1], pieces[1:]):
        pa, pb = samples[a.sample].positions[a.hi - 1], samples[b.sample].positions[b.lo]
        assert (pb['major'], pb['minor']) in ((pa['major'] + 1, 0), (pa['major'], pa['minor'] + 1))


def test_fill_gaps_and_fastx(tmp_path):
    draft = {"r1": "ACGTACGTACGTACGTACGT", "r2": "TTTTTTTTTT"}
    contigs = [(("r1", 2, 5), ["gg", "g"], ["##", "#"]), (("r1", 10, 14), ["ccccc"], ["$$$$$"]),
               (("r2", 0, 9), ["AAAAAAAAAA"], ["%%%%%%%%%%"])]
    filled, gaps = stitch.fill_gaps(contigs, draft)
    assert [c[0] for c in filled] == [("r1", 0, 20), ("r2", 0, 10)]
    assert ''.join(filled[0][1]) == "AC" + "ggg" + "GTAC" + "ccccc" + "TACGT"
    assert ''.join(filled[0][2]) == "!!" + "###" + "!!!!" + "$$$$$" + "!!!!!"
    assert gaps == {"r1": [(0, 2), (6, 10), (15, 20)], "r2": []}
    filled_n, _ = stitch.fill_gaps(contigs, draft, fill_char="N")
    assert ''.join(filled_n[0][1]) == "NN" + "ggg" + "NNNN" + "ccccc" + "NNNNN"
    buf = io.StringIO()
    stitch.write_fastx_segment(buf, ("r2", filled[1][1], filled[1][2]), qualities=True)
    stitch.write_fastx_segment(buf, ("r2", filled[1][1], filled[1][2]), qualities=False)
    assert buf.getvalue() == "@r2\nAAAAAAAAAA\n+\n%%%%%%%%%%\n>r2\nAAAAAAAAAA\n"
    fa = tmp_path / "d.fa"
    fa.write_text(">r1 some description\nACGTACGTAC\nGTACGTACGT\n>r2\nTTTTTTTTTT\n")
    assert dict(stitch.read_fasta(str(fa))) == draft


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_gpu_stitch_matches_reference(golden_dir):
    for name, rec in _golden(golden_dir).items():
        samples = _samples(synth.synth_stitch_stream(**rec["kwargs"]))
        got = stitch.stitch_samples(samples, None, Region('contig1', rec["start"], rec["end"]), rec["min_depth"])
        assert _flatten(got) == rec["contigs"], name


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [[1], [3], [4], [5], [1023], [1024], [1025], [7, 1, 1, 2050, 3, 1021],
                                  [4096, 4096], [100003]])
def test_gpu_decode_pieces_shapes(rows):
    """Block / vector-width boundaries, one-row ranges, many ranges in one 4-row group; phred edges first in each range."""
    rs = np.random.RandomState(sum(rows))
    samples, pieces = [], []
    for k, n in enumerate(rows):
        p = rs.dirichlet(np.ones(5) * 0.3, size=n + 6).astype(np.float32)
        p[rs.rand(n + 6) < 0.4] = np.array([0.9, 0.025, 0.025, 0.025, 0.025], np.float32)      # gap calls
        m = min(n, len(PHRED_EDGE_P))
        p[3:3 + m] = phred_edge_rows()[:m]
        samples.append(Sample('c', None, None, None, None, p, None))
        pieces.append(stitch.Piece(k, 3, 3 + n, False, False))
    seqs, quals = stitch.decode_pieces(samples, pieces)
    exp_s, exp_q = _cpu_decode(samples, pieces)
    assert seqs == exp_s and quals == exp_q
    seqs_only, none = stitch.decode_pieces(samples, pieces, with_qualities=False)
    assert seqs_only == exp_s and none is None


@pytest.mark.gpu
def test_gpu_decode_pieces_degenerate():
    allgap = np.tile(np.array([0.6, 0.1, 0.1, 0.1, 0.1], np.float32), (5000, 1))
    nogap = np.tile(np.array([0.0, 0.0, 1.0, 0.0, 0.0], np.float32), (5000, 1))
    ties = np.tile(np.array([0.2, 0.2, 0.2, 0.2, 0.2], np.float32), (9, 1))        # first maximum (gap) wins
    ties2 = np.tile(np.array([0.1, 0.3, 0.3, 0.2, 0.1], np.float32), (9, 1))       # -> 'A'
    samples = [Sample('c', None, None, None, None, x, None) for x in (allgap, nogap, ties, ties2)]
    pieces = [stitch.Piece(k, 0, len(samples[k].label_probs), False, False) for k in range(4)]
    seqs, quals = stitch.decode_pieces(samples, pieces)
    assert seqs == ["", "C" * 5000, "", "A" * 9]
    assert quals[1] == chr(33 + 70) * 5000 and quals[0] == "" and len(quals[3]) == 9
    assert stitch.decode_pieces(samples, []) == ([], [])
    with pytest.raises(ValueError):
        stitch.decode_pieces([Sample('c', None, None, None, None, np.zeros((4, 4), np.float32), None)],
                             [stitch.Piece(0, 0, 4, False, False)])


@pytest.mark.gpu
def test_gpu_stitch_large_vs_oracle():
    """~1.2e6 columns in 130 samples with every perturbation; bytes identical to the CPU restatement."""
    kw = dict(seed=21, n_major=1_000_000, chunk_len=10_000, overlap=1_000, p_ins=0.15, ragged=(3, 40, 77),
              drop=(10, 90), nest=(20, 60), low_depth=((5, 4000, 4100), (50, 9000, 9500)))
    stream = synth.synth_stitch_stream(**kw)
    exp = stitch_oracle.stitch_samples(stream, 5000, 990_000, 10)
    got = stitch.stitch_samples(_samples(stream), None, Region('contig1', 5000, 990_000), 10)
    assert _flatten(got) == _flatten(exp)
    assert len(got) >= 5
