"""The CPU oracle against the reference binary's outputs on reads at the ends of reference sequences (tests/golden/synth_edges,
make_golden_edges.sh): one 60 kbp sequence and 50 short ones (20 bp to 3 kbp), 70% of the fragments within 40 bp of a
sequence's start or end.  Every file byte for byte; and each BED must hold enough records at the edges to show they were reached.
CPU only."""
import gzip
import hashlib
import os

import pytest

from oracle import oracle_py as orc
from tests.util import read_fasta

# name -> (preset, knobs, paired, error threshold)
EDGE_CASES = {
    "chip.bed": ("chip", {}, True, 8),
    "q0.bed": ("", dict(mapq_threshold=0), True, 8),
    "e15q0.bed": ("", dict(error_threshold=15, mapq_threshold=0), True, 15),
    "e1q0.bed": ("", dict(error_threshold=1, mapq_threshold=0), True, 1),
    "atac.bed": ("atac", {}, True, 8),
    "se_q0.bed": ("", dict(mapq_threshold=0), False, 8),
    "pe_q0.sam": ("", dict(mapq_threshold=0), True, 8),
    "se_q0.sam": ("", dict(mapq_threshold=0), False, 8),
    "hic_q0.pairs": ("hic", dict(mapq_threshold=0), True, 8),
}


def _spans(text):
    """(sequence name, start, end) of every record of BED, SAM or pairs text, 0-based, end exclusive; for pairs, each mate's
    5' position as a one-base span."""
    for line in text.splitlines():
        if line[:1] in (b"@", b"#"):
            continue
        f = line.split(b"\t")
        if len(f) > 10:   # SAM: POS is 1-based, the CIGAR's M / D / N / = / X operations span the reference
            st, num, ref_len = int(f[3]) - 1, 0, 0
            for c in f[5]:
                if 48 <= c <= 57:
                    num = num * 10 + c - 48
                else:
                    ref_len += num if c in b"MDN=X" else 0
                    num = 0
            yield f[2].decode(), st, st + ref_len
        elif len(f) >= 7 and f[6] in (b"+", b"-"):   # pairs: readID chr1 pos1 chr2 pos2 strand1 strand2 (1-based)
            yield f[1].decode(), int(f[2]) - 1, int(f[2])
            yield f[3].decode(), int(f[4]) - 1, int(f[4])
        else:
            yield f[0].decode(), int(f[1]), int(f[2])


def edge_counts(text, seq_len, read_len, e):
    """(records starting within L + e of the start of a sequence other than the first, records ending within e + 1 of their
    sequence's end, records on sequences shorter than 2L) of BED, SAM or pairs text; seq_len: name -> length."""
    first = next(iter(seq_len))
    start = end = short = 0
    for name, st, en in _spans(text):
        start += name != first and st < read_len + e
        end += en + e + 1 >= seq_len[name]
        short += seq_len[name] < 2 * read_len
    return start, end, short


# name -> at least (records starting within L + e of a sequence other than the first, ending within e + 1 of a sequence's end, on
# sequences shorter than 2L).  At -e 15 only the 90 and 99 bp sequences are both shorter than 2L and longer than L + 2e; --preset
# atac shifts the ends of its records (Tn5) away from the sequence ends.
EDGE_FLOORS = {"chip.bed": (570, 24, 25), "q0.bed": (600, 26, 28), "e15q0.bed": (430, 11, 3), "e1q0.bed": (740, 24, 100), "atac.bed": (560, 0, 25),
               "se_q0.bed": (390, 14, 55), "pe_q0.sam": (660, 27, 55), "se_q0.sam": (390, 14, 55), "hic_q0.pairs": (295, 30, 36)}


def assert_reaches_the_edges(case, text, seq_len):
    preset, _, _, e = EDGE_CASES[case]
    got = edge_counts(text, seq_len, 150 if preset == "hic" else 50, e)
    assert all(g >= f for g, f in zip(got, EDGE_FLOORS[case])), (case, got, EDGE_FLOORS[case])


@pytest.fixture(scope="module")
def edges(golden_dir, tmp_path_factory):
    d = os.path.join(golden_dir, "synth_edges")
    ref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    p = str(tmp_path_factory.mktemp("edges") / "ref.index")
    assert orc.Index(ref=ref, k=17, w=7).save(p) == 0
    md5 = dict(reversed(line.split()) for line in open(os.path.join(d, "md5.txt")))
    names, seqs = read_fasta(os.path.join(d, "ref.fa.gz"))
    return dict(d=d, index=p, md5=md5, seq_len={n: len(s) for n, s in zip(names, seqs)})


@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_oracle_reproduces_reference_binary_at_sequence_ends(edges, tmp_path, case):
    preset, kw, paired, _ = EDGE_CASES[case]
    d = edges["d"]
    p = orc.make_params(preset, **kw)
    out = str(tmp_path / case)
    ref = os.path.join(d, "ref.fa.gz")
    r1, r2 = (os.path.join(d, "hic_read1.fq.gz"), os.path.join(d, "hic_read2.fq.gz")) if preset == "hic" else \
        (os.path.join(d, "read1.fq.gz"), os.path.join(d, "read2.fq.gz"))
    if case.endswith(".sam"):
        orc.run_files_sam(p, edges["index"], ref, r1, r2 if paired else None, out)
    elif paired:
        orc.run_files(p, edges["index"], ref, r1, r2, out)
    else:
        orc.run_files_se(p, edges["index"], ref, r1, out, 1)
    want = gzip.open(os.path.join(d, case + ".gz")).read()
    assert hashlib.md5(want).hexdigest() == edges["md5"][case]
    assert open(out, "rb").read() == want
    assert_reaches_the_edges(case, want, edges["seq_len"])
