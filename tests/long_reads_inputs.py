"""Seeded read sets longer than 160 bases on synth_sc's reference (3 sequences, 750 kbp), for tests/golden/synth_long
(make_golden_long.sh) and the GPU tests of reads beyond the default `max_read_length`.

Fragments are drawn uniformly from the reference, both strands, with about 1 % substitutions, a few one-base indels and N's.
Kinds:
  pe<L>   pairs of L-base mates, fragments of max(L - 60, L / 2) .. 3L bases: the shortest read into the Nextera adapter, which
          `--preset atac` trims;
  mixed   pairs whose mates are 50 .. 300 bases each, independently; mixed<M>: 50 .. M bases;
  se<L>   read 1 of pe<L>;
  hic<L>  Hi-C-like pairs: mates from two loci, a third of read 1 chimeric (its tail from read 2's locus).
Barcodes (`barcodes`) are drawn from synth_sc's whitelist, one in ten with one substitution."""
import gzip
import os

import numpy as np

from tests.util import read_fasta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "synth_sc", "ref.fa.gz")
WHITELIST = os.path.join(ROOT, "tests", "golden", "synth_sc", "whitelist.txt")
ADAPTER = b"CTGTCTCTTATACACATCTCCGAGCCCACGAGACTAAGGCGAATCTCGTATGCCGTCTTCTGCTTG"
COMP = bytes.maketrans(b"ACGTN", b"TGCAN")


def _mutate(g, s):
    s = bytearray(s)
    for i in np.nonzero(g.random(len(s)) < 0.01)[0]:
        s[i] = b"ACGT"[g.integers(4)]
    if g.random() < 0.15:  # a one-base insertion or deletion
        i = int(g.integers(10, len(s) - 10))
        s[i:i + 1] = b"" if g.random() < 0.5 else bytes([s[i], b"ACGT"[g.integers(4)]])
    if g.random() < 0.05:
        s[int(g.integers(len(s)))] = ord("N")
    return bytes(s)


def _frag(g, seqs, n):
    """n bases from a random place of a random sequence (long enough), on a random strand."""
    while True:
        r = int(g.integers(len(seqs)))
        if len(seqs[r]) > n + 2:
            break
    p = int(g.integers(0, len(seqs[r]) - n))
    f = seqs[r][p:p + n].tobytes()
    return f.translate(COMP)[::-1] if g.random() < 0.5 else f


def _mate(g, frag, L):
    """The first L bases of a fragment, read into the adapter when the fragment is shorter."""
    s = frag[:L]
    if len(s) < L:
        s += (ADAPTER + bytes(g.choice(list(b"ACGT"), size=L)))[:L - len(s)]
    return _mutate(g, s)


def make_pairs(kind, n, seed, seqs=None):
    """[(read 1, read 2)] of one kind (read 2 None for single-end), from synth_sc's reference or the sequences given."""
    g = np.random.default_rng(seed)
    if seqs is None:
        _, seqs = read_fasta(REF)
    out = []
    for _ in range(n):
        if kind.startswith("mixed"):
            hi = int(kind[5:] or 300)
            l1, l2 = int(g.integers(50, hi + 1)), int(g.integers(50, hi + 1))
            f = _frag(g, seqs, int(g.integers(max(l1, l2), 3 * max(l1, l2) + 1)))
            out.append((_mutate(g, f[:l1]), _mutate(g, f.translate(COMP)[::-1][:l2])))
        elif kind.startswith("hic"):
            L = int(kind[3:])
            a, b = _frag(g, seqs, L), _frag(g, seqs, L)
            if g.random() < 1 / 3:
                cut = int(g.integers(L // 3, 2 * L // 3))
                a = a[:cut] + b.translate(COMP)[::-1][:L - cut]
            out.append((_mutate(g, a), _mutate(g, b)))
        else:
            L = int(kind[2:])
            f = _frag(g, seqs, int(g.integers(max(L - 60, L // 2), 3 * L + 1)))
            r1, r2 = _mate(g, f, L), _mate(g, f.translate(COMP)[::-1], L)
            out.append((r1, None if kind.startswith("se") else r2))
    return out


def barcodes(n, seed):
    g = np.random.default_rng(seed)
    wl = [l.strip().encode() for l in open(WHITELIST) if l.strip()]
    out = []
    for _ in range(n):
        b = bytearray(wl[int(g.integers(len(wl)))])
        if g.random() < 0.1:
            b[int(g.integers(len(b)))] = b"ACGT"[g.integers(4)]
        out.append(bytes(b))
    return out


def write_fastq(path, reads, prefix):
    with (gzip.GzipFile(path, "wb", mtime=0) if path.endswith(".gz") else open(path, "wb")) as f:
        for i, r in enumerate(reads):
            f.write(b"@%s%d\n%s\n+\n%s\n" % (prefix.encode(), i, r, b"I" * len(r)))


def write_set(d, kind, n, seed, tag=None):
    """read1 / read2 FASTQ files of one kind under d: <tag>_1.fq.gz, <tag>_2.fq.gz (single-end: _1 only)."""
    tag = tag or kind
    pairs = make_pairs(kind, n, seed)
    p1 = os.path.join(d, tag + "_1.fq.gz")
    write_fastq(p1, [a for a, _ in pairs], tag + ".")
    if pairs[0][1] is None:
        return p1, None
    p2 = os.path.join(d, tag + "_2.fq.gz")
    write_fastq(p2, [b for _, b in pairs], tag + ".")
    return p1, p2


# the golden inputs: kind -> (pairs, seed)
GOLDEN_SETS = {"pe250": (5000, 250), "pe300": (4000, 300), "mixed": (5000, 77), "se250": (5000, 251), "hic250": (4000, 252)}
# reads beyond 320 bases, written where a test runs (the reference binary maps them there): kind -> (pairs, seed)
BEYOND_320_SETS = {"pe400": (2000, 400), "pe600": (1500, 600), "pe832": (1000, 832), "mixed1400": (1500, 1400), "se600": (1500, 601), "hic400": (1500, 402)}


if __name__ == "__main__":
    import sys
    d = sys.argv[1]
    for kind, (n, seed) in GOLDEN_SETS.items():
        write_set(d, kind, n, seed)
    write_fastq(os.path.join(d, "barcode.fq.gz"), barcodes(GOLDEN_SETS["pe250"][0], 16), "pe250.")
