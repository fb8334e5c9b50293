#!/usr/bin/env python
"""Synthetic reference + paired-end read generator (SURVEY.md §8(d) configs, scaled).

Writes ref.fa, read1.fq, read2.fq (optionally barcode.fq) into --out.  Deterministic for a seed.
Used by tests (small sizes), by oracle pinning against the compiled reference binary, and by
bench.py's cpu_baseline / --impl reference legs (bounded samples).  numpy only.
"""
import argparse
import os
import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
COMP[:] = ord("N")
for a, b in zip(b"ACGTacgt", b"TGCAtgca"):
    COMP[a] = b
ADAPTER1 = np.frombuffer(b"CTGTCTCTTATACACATCTCCGAGCCCACGAGAC" * 8, dtype=np.uint8)
ADAPTER2 = np.frombuffer(b"CTGTCTCTTATACACATCTGACGCTGCCGACGA" * 8, dtype=np.uint8)


def make_reference(rng, n_seq, seq_len, repeat_len=5000, repeat_copies=50, fam_len=300,
                   fam_copies=0, n_frac=0.001, lowercase_frac=0.0):
    seqs = []
    fam = ACGT[rng.integers(0, 4, fam_len)]
    for _ in range(n_seq):
        s = ACGT[rng.integers(0, 4, seq_len)].copy()
        # planted segmental repeat: one segment, `repeat_copies` copies (half exact, half 1% diverged)
        if repeat_copies > 0 and seq_len > 4 * repeat_len * repeat_copies // 3:
            seg = ACGT[rng.integers(0, 4, repeat_len)]
            starts = rng.integers(0, seq_len - repeat_len, repeat_copies)
            for ci, st in enumerate(starts):
                c = seg.copy()
                if ci % 2 == 1:
                    m = rng.random(repeat_len) < 0.01
                    c[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
                s[st:st + repeat_len] = c
        # short high-copy family (exercises the f=500/1000 frequency caps)
        if fam_copies > 0:
            starts = rng.integers(0, seq_len - fam_len, fam_copies)
            for st in starts:
                c = fam.copy()
                m = rng.random(fam_len) < 0.005
                c[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
                s[st:st + fam_len] = c
        # N runs
        n_target = int(seq_len * n_frac)
        while n_target > 0:
            ln = int(rng.integers(1, 200))
            st = int(rng.integers(0, max(1, seq_len - ln)))
            s[st:st + ln] = ord("N")
            n_target -= ln
        if lowercase_frac > 0:
            n_lc = int(seq_len * lowercase_frac / 500)
            for st in rng.integers(0, max(1, seq_len - 500), n_lc):
                seg = s[st:st + 500]
                isb = (seg != ord("N")) & (seg < 97)
                seg[isb] = seg[isb] + 32
        seqs.append(s)
    return seqs


def mutate(rng, frag, sub_rate, indel_rate):
    """Apply substitutions and (rarely) single-base indels to a fragment end (returns new array)."""
    out = frag.copy()
    if sub_rate > 0:
        m = rng.random(len(out)) < sub_rate
        k = int(m.sum())
        if k:
            out[m] = ACGT[rng.integers(0, 4, k)]
    if indel_rate > 0 and rng.random() < indel_rate * len(out):
        p = int(rng.integers(1, len(out) - 1))
        if rng.random() < 0.5:
            out = np.concatenate([out[:p], ACGT[rng.integers(0, 4, 1)], out[p:]])
        else:
            out = np.concatenate([out[:p], out[p + 1:]])
    return out


def revcomp(a):
    return COMP[a[::-1]]


def make_short_seqs(rng, n):
    """n short sequences, as in a scaffold-level assembly: lengths where the mapping rules change for 2x50 and 2x150 reads at
    -e 8 and 15 (below k + w - 1, around L + 2e, around a fragment), then a spread up to 3 kbp."""
    lens = [20, 30, 60, 70, 75, 80, 90, 99, 100, 101, 120, 150, 180, 250][:n]
    lens += [int(x) for x in rng.integers(300, 3001, n - len(lens))]
    return [ACGT[rng.integers(0, 4, ln)].copy() for ln in lens]


def make_reads(rng, seqs, n_pairs, read_len, frag_min=80, frag_max=500, sub_rate=0.01,
               indel_rate=0.001, dup_frac=0.05, short_frac=0.0, n_read_frac=0.002,
               junk_frac=0.01, chimeric_frac=0.0, edge_frac=0.0, edge_rng=None):
    """Returns list of (r1, r2) uint8 arrays.  A fraction edge_frac of the fragments (drawn from edge_rng) starts within 40 bp of
    a sequence's start or ends within 40 bp of its end, on any sequence; a fragment longer than its sequence is cut to it."""
    pairs = []
    n_seq = len(seqs)
    lens = np.array([len(s) for s in seqs])
    frags = []
    while len(pairs) < n_pairs:
        if frags and rng.random() < dup_frac:
            si, st, fl, strand = frags[int(rng.integers(0, len(frags)))]
        else:
            si = int(rng.integers(0, n_seq))
            if short_frac > 0 and rng.random() < short_frac:
                fl = int(rng.integers(32, 100))
            else:
                fl = int(rng.integers(frag_min, frag_max + 1))
            if edge_frac > 0 and edge_rng.random() < edge_frac:
                si = int(edge_rng.integers(0, n_seq))
                if fl > lens[si]:
                    fl = int(edge_rng.integers(min(read_len, lens[si]), lens[si] + 1))
                d = int(edge_rng.integers(0, min(40, lens[si] - fl) + 1))
                st = d if edge_rng.random() < 0.5 else int(lens[si]) - fl - d
            elif lens[si] > fl:
                st = int(rng.integers(0, lens[si] - fl))
            else:
                st, fl = 0, int(lens[si])
            strand = int(rng.integers(0, 2))
            frags.append((si, st, fl, strand))
            if len(frags) > 4096:
                frags.pop(int(rng.integers(0, len(frags))))
        if rng.random() < junk_frac:
            r1 = ACGT[rng.integers(0, 4, read_len)]
            r2 = ACGT[rng.integers(0, 4, read_len)]
            pairs.append((r1, r2))
            continue
        frag = seqs[si][st:st + fl]
        fwd = frag
        rev = revcomp(frag)
        if strand:
            fwd, rev = rev, fwd
        # read-through into adapter when the fragment is shorter than the read
        e1 = np.concatenate([fwd, ADAPTER1])[:read_len + 4]
        e2 = np.concatenate([rev, ADAPTER2])[:read_len + 4]
        r1 = mutate(rng, e1, sub_rate, indel_rate)[:read_len]
        r2 = mutate(rng, e2, sub_rate, indel_rate)[:read_len]
        if chimeric_frac > 0 and rng.random() < chimeric_frac:
            # ligation junction: tail of r1 comes from an independent locus
            j = int(rng.integers(30, max(31, read_len - 30)))
            sj = int(rng.integers(0, n_seq))
            if lens[sj] <= read_len:
                sj = 0
            pj = int(rng.integers(0, lens[sj] - read_len))
            other = seqs[sj][pj:pj + read_len - j]
            if rng.random() < 0.5:
                other = revcomp(other)
            r1 = np.concatenate([r1[:j], other])[:read_len]
        if rng.random() < n_read_frac:
            r1 = r1.copy()
            r1[int(rng.integers(0, len(r1)))] = ord("N")
        # upper-case reads (sequencers emit upper case); reference may be soft-masked
        r1 = np.where(r1 >= 97, r1 - 32, r1).astype(np.uint8)
        r2 = np.where(r2 >= 97, r2 - 32, r2).astype(np.uint8)
        pairs.append((r1, r2))
    return pairs


def write_fasta(path, seqs, names=None):
    with open(path, "wb") as f:
        for i, s in enumerate(seqs):
            nm = names[i] if names else "chr%d" % (i + 1)
            f.write(b">" + nm.encode() + b" synthetic\n")
            b = s.tobytes()
            for j in range(0, len(b), 80):
                f.write(b[j:j + 80] + b"\n")


def write_fastq(path, reads, prefix, suffix):
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b"@%s.%d/%s\n" % (prefix.encode(), i, suffix.encode()))
            f.write(r.tobytes() + b"\n+\n" + b"I" * len(r) + b"\n")


def make_barcodes(rng, n_pairs, n_whitelist=2000, n_cells=200, bc_len=16, err_frac=0.02):
    wl = ACGT[rng.integers(0, 4, (n_whitelist, bc_len))]
    wl = np.unique(wl, axis=0)
    cells = wl[rng.integers(0, len(wl), n_cells)]
    bcs = cells[rng.integers(0, n_cells, n_pairs)].copy()
    quals = rng.integers(2, 41, (n_pairs, bc_len)).astype(np.uint8) + 33
    m = rng.random(n_pairs) < err_frac
    idx = np.nonzero(m)[0]
    pos = rng.integers(0, bc_len, len(idx))
    bcs[idx, pos] = ACGT[rng.integers(0, 4, len(idx))]
    return wl, bcs, quals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--n-seq", type=int, default=4)
    ap.add_argument("--seq-len", type=int, default=1_000_000)
    ap.add_argument("--n-pairs", type=int, default=20000)
    ap.add_argument("--read-len", type=int, default=50)
    ap.add_argument("--repeat-copies", type=int, default=50)
    ap.add_argument("--repeat-len", type=int, default=5000)
    ap.add_argument("--fam-copies", type=int, default=1500)
    ap.add_argument("--short-frac", type=float, default=0.0)
    ap.add_argument("--chimeric-frac", type=float, default=0.0)
    ap.add_argument("--lowercase-frac", type=float, default=0.0)
    ap.add_argument("--barcodes", action="store_true")
    # edge-heavy inputs (own generator: every other set stays as it was)
    ap.add_argument("--short-seqs", type=int, default=0, help="short sequences after the --n-seq long ones")
    ap.add_argument("--edge-frac", type=float, default=0.0, help="fraction of fragments at the ends of sequences")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    rng = np.random.default_rng(a.seed)
    seqs = make_reference(rng, a.n_seq, a.seq_len, a.repeat_len, a.repeat_copies,
                          fam_copies=a.fam_copies, lowercase_frac=a.lowercase_frac)
    edge_rng = np.random.default_rng([a.seed, 1])
    seqs += make_short_seqs(edge_rng, a.short_seqs)
    write_fasta(os.path.join(a.out, "ref.fa"), seqs)
    pairs = make_reads(rng, seqs, a.n_pairs, a.read_len, short_frac=a.short_frac,
                       chimeric_frac=a.chimeric_frac, edge_frac=a.edge_frac, edge_rng=edge_rng)
    write_fastq(os.path.join(a.out, "read1.fq"), [p[0] for p in pairs], "r", "1")
    write_fastq(os.path.join(a.out, "read2.fq"), [p[1] for p in pairs], "r", "2")
    if a.barcodes:
        wl, bcs, quals = make_barcodes(rng, a.n_pairs)
        with open(os.path.join(a.out, "whitelist.txt"), "wb") as f:
            for w in wl:
                f.write(w.tobytes() + b"\n")
        with open(os.path.join(a.out, "barcode.fq"), "wb") as f:
            for i in range(a.n_pairs):
                f.write(b"@r.%d\n" % i + bcs[i].tobytes() + b"\n+\n" + quals[i].tobytes() + b"\n")


if __name__ == "__main__":
    main()
