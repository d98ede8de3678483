"""Host side of `medaka sequence` over this package's stores (stitch.sequence / stitch.write_consensus): the sample
index, the stitch regions, sample selection at region boundaries, verbatim contigs, the gap bed and the record names
without gap filling.  Decoding is replaced by a host stand-in, so no GPU is needed."""
import os

import numpy as np

from medaka_b200 import common, stitch


def _positions(majors, minors):
    return np.array(list(zip(majors, minors)), dtype=[("major", np.int64), ("minor", np.int64)])


def _sample(ref, first, last):
    """A sample covering majors first .. last (one major column each)."""
    majors = np.arange(first, last + 1)
    return common.Sample(ref_name=ref, features=None, labels=None, ref_seq=None,
                         positions=_positions(majors, np.zeros_like(majors)), label_probs=None,
                         depth=np.full(len(majors), 10))


def _fake_decode(samples, pieces):
    # base = 'ACGT'[major % 4], quality = chr(33 + major % 40): what each row was is visible in the output
    seqs, quals = [], []
    for p in pieces:
        m = samples[p.sample].positions["major"][p.lo:p.hi]
        seqs.append("".join("ACGT"[int(x) % 4] for x in m))
        quals.append("".join(chr(33 + int(x) % 40) for x in m))
    return seqs, quals


def test_index_orders_by_start_then_longest_first():
    names = ["b:10.0-20.0", "b:10.0-30.0", "b:10.1-15.0", "a:5.0-9.0", "b:2.3-4.0", "b:100.0-120.0", "b:20.0-25.0",
             "b:10.0-30.2", "not a sample name"]
    index = stitch.sample_index(names)
    assert list(index) == ["a", "b"]
    assert index["a"] == ["a:5.0-9.0"]
    # majors compare as numbers (100 after 20), then minors; equal starts: the later end first
    assert index["b"] == ["b:2.3-4.0", "b:10.0-30.2", "b:10.0-30.0", "b:10.0-20.0", "b:10.1-15.0", "b:20.0-25.0",
                          "b:100.0-120.0"]


def test_regions_split_at_one_megabase_and_missing_contigs():
    index = {"long": [], "short": []}
    lengths = {"long": 2500000, "short": 700, "absent": 50}
    todo, missing = stitch.plan_regions(index, lengths)
    R = common.Region
    assert todo == [R("long", 0, 1000000), R("long", 1000000, 2000000), R("long", 2000000, 2500000),
                    R("short", 0, 700)]
    assert missing == ["absent"]
    todo, missing = stitch.plan_regions(index, lengths, ["long:500000-1700000", R("short", 100, None), "absent",
                                                         "absent:0-10"])
    assert todo == [R("long", 500000, 1500000), R("long", 1500000, 1700000), R("short", 100, 700)]
    assert missing == ["absent"]


def test_selection_at_region_boundaries():
    names = ["c:990000.0-999999.3", "c:995000.0-1000000.2", "c:1000000.0-1009000.0", "c:1999999.1-2000000.0",
             "d:0.0-10.0"]
    index = stitch.sample_index(names)
    R = common.Region
    # a sample covers [int(start major), int(end major) + 1)
    assert stitch.select_samples(index, R("c", 0, 1000000)) == names[:2]
    assert stitch.select_samples(index, R("c", 1000000, 2000000)) == names[1:4]
    assert stitch.select_samples(index, R("c", 2000000, 3000000)) == [names[3]]
    assert stitch.select_samples(index, R("e", 0, 10)) == []


def _run(tmp_path, samples, draft, **kw):
    by_name = {s.name: s for s in samples}
    out = str(tmp_path / "out.fastq")
    stitch.write_consensus(stitch.sample_index(by_name), lambda names: [by_name[n] for n in names], draft, out,
                           decode=_fake_decode, **kw)
    with open(out) as fh:
        text = fh.read()
    bed = out + ".gaps_in_draft_coords.bed"
    bed_text = None
    if os.path.exists(bed):
        with open(bed) as fh:
            bed_text = fh.read()
    return text, bed_text


def test_fillgaps_bed_and_verbatim_contigs(tmp_path):
    draft = {"z": "N" * 30, "a": "ACGTACGTAC" * 5, "m": "TTTT"}
    samples = [_sample("a", 5, 19), _sample("a", 15, 24), _sample("a", 40, 44)]
    text, bed = _run(tmp_path, samples, draft)
    seq = "".join("ACGT"[m % 4] for m in range(5, 25))
    qual = "".join(chr(33 + m % 40) for m in range(5, 25))
    tail = "".join("ACGT"[m % 4] for m in range(40, 45))
    tail_q = "".join(chr(33 + m % 40) for m in range(40, 45))
    a = draft["a"]
    expect_a = a[:5] + seq + a[25:40] + tail + a[45:]
    expect_aq = "!" * 5 + qual + "!" * 15 + tail_q + "!" * 5
    # contigs with samples first, in request (draft) order, then the verbatim ones
    assert text == "@a\n{}\n+\n{}\n@z\n{}\n+\n{}\n@m\nTTTT\n+\n!!!!\n".format(
        expect_a, expect_aq, draft["z"], "!" * 30)
    assert bed == "a\t0\t5\na\t25\t40\na\t45\t50\nm\t0\t4\nz\t0\t30\n"
    # FASTA and a fill character
    text, _ = _run(tmp_path, samples, draft, qualities=False, fill_char="x", regions=["a"])
    assert text == ">a\n{}\n".format("x" * 5 + seq + "x" * 15 + tail + "x" * 5)


def test_no_fillgaps_names_pieces_per_contig(tmp_path):
    draft = {"a": "A" * 100, "b": "C" * 100}
    samples = [_sample("a", 5, 19), _sample("a", 40, 44), _sample("b", 0, 9), _sample("b", 10, 12)]
    text, bed = _run(tmp_path, samples, draft, fillgaps=False, qualities=False)
    assert bed is None
    names = [line[1:] for line in text.splitlines() if line.startswith(">")]
    # abutting samples of b collapse into one record
    assert names == ["a_0 5-20", "a_1 40-45", "b_0 0-13"]


def test_min_depth_and_region_subset(tmp_path):
    draft = {"a": "G" * 60}
    s = _sample("a", 0, 49)
    depth = np.full(50, 10)
    depth[20:30] = 1
    s = s.amend(depth=depth)
    text, bed = _run(tmp_path, [s], draft, fillgaps=False, min_depth=5, regions=["a:10-40"])
    names = [line[1:] for line in text.splitlines() if line.startswith("@")]
    assert names == ["a_0 10-20", "a_1 30-40"]
