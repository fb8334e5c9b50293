#!/usr/bin/env python
"""Reads and a reference beyond upper-case ACGTN, for tests/golden/synth_bytes (make_golden_bytes.sh).  Deterministic for a seed.

The reference: three sequences (300 kbp), a 300 bp family with many copies and a 2 kbp segmental repeat (multi-mappers, the
overflow tiers), N runs, soft-masked stretches of 50 to 2,000 bases over about 40 % of it, IUPAC codes in both cases and a
sprinkling of bytes 0x80-0xFF (a third of them at 0xE0-0xFF).  Lines end in LF; no line starts with '>', '+' or '@'.

The reads: 2x100 (a third of the fragments shorter than the reads: adapter read-through), 2x150 Hi-C with a ligation junction
in half of read 1, 2x250.  Each mate carries one decoration: none, wholly lower case, lower-case runs, lower-case 'n', '.',
IUPAC codes, or (read taken from the forward strand) every reference byte of 0x80 and above copied 32 lower, so that it sits
opposite the reference byte it matches under the signed rule of the Hi-C gap extension.  Fragments keep 50 bases from the ends
of their sequence.

--normalise writes the same inputs with every byte the reference's CharToUint8 maps to 0..3 as its upper-case base and every
other byte as 'N' (the index and the case-folded mapping do not change; only the effects of the raw bytes go away)."""
import argparse
import os

import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
IUPAC = np.frombuffer(b"RYKMSWBDHVrykmswbdhv", dtype=np.uint8)
COMP = np.full(256, ord("N"), dtype=np.uint8)
for a, b in zip(b"ACGTacgt", b"TGCAtgca"):
    COMP[a] = b
# CharToUint8 (utils.h): A/a C/c G/g T/t -> 0..3, every other byte -> 4
NORMALISE = np.full(256, ord("N"), dtype=np.uint8)
for a, b in zip(b"ACGTacgt", b"ACGTACGT"):
    NORMALISE[a] = b
ADAPTER1 = np.frombuffer(b"CTGTCTCTTATACACATCTCCGAGCCCACGAGAC" * 8, dtype=np.uint8)
ADAPTER2 = np.frombuffer(b"CTGTCTCTTATACACATCTGACGCTGCCGACGA" * 8, dtype=np.uint8)
DECORATIONS = ("none", "lower", "lower_runs", "lower_n", "dot", "iupac", "high")


def make_reference(rng, lens=(120000, 100000, 80000)):
    fam = ACGT[rng.integers(0, 4, 300)]
    seg = ACGT[rng.integers(0, 4, 2000)]
    seqs = []
    for n in lens:
        s = ACGT[rng.integers(0, 4, n)].copy()
        for st in rng.integers(100, n - 2100, 6):   # segmental repeat, half of the copies 1 % diverged
            c = seg.copy()
            if rng.random() < 0.5:
                m = rng.random(len(c)) < 0.01
                c[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
            s[st:st + 2000] = c
        for st in rng.integers(100, n - 400, 60):     # 300 bp family, 0.5 % diverged copies
            c = fam.copy()
            m = rng.random(300) < 0.005
            c[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
            s[st:st + 300] = c
        for _ in range(8):                            # N runs
            ln = int(rng.integers(1, 300))
            st = int(rng.integers(0, n - ln))
            s[st:st + ln] = ord("N")
        masked = np.zeros(n, dtype=bool)              # soft-masked stretches of 50 to 2,000 bases, about 40 %
        while masked.mean() < 0.4:
            ln = int(rng.integers(50, 2001))
            st = int(rng.integers(0, n - ln))
            masked[st:st + ln] = True
        s[masked] = np.where((s[masked] >= 65) & (s[masked] <= 90), s[masked] + 32, s[masked])
        pos = rng.choice(n, n // 400, replace=False)  # IUPAC codes, upper and lower case
        s[pos] = IUPAC[rng.integers(0, len(IUPAC), len(pos))]
        pos = rng.choice(n, n // 120, replace=False)  # bytes 0x80-0xFF: a third each at 0x80-0x9F, 0xA0-0xDF, 0xE0-0xFF
        band = rng.integers(0, 3, len(pos))
        s[pos] = (np.array([0x80, 0xA0, 0xE0])[band] + rng.integers(0, np.array([32, 64, 32])[band])).astype(np.uint8)
        seqs.append(s)
    return seqs


def mutate(rng, r, sub_rate=0.01, indel_rate=0.001):
    out = r.copy()
    m = rng.random(len(out)) < sub_rate
    out[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
    if rng.random() < indel_rate * len(out):
        p = int(rng.integers(1, len(out) - 1))
        out = np.concatenate([out[:p], ACGT[rng.integers(0, 4, 1)], out[p:]]) if rng.random() < 0.5 else np.concatenate([out[:p], out[p + 1:]])
    return out


def sequenced(rng, raw):
    """What a sequencer reads off a reference stretch: upper-case ACGT, a random base where the reference has no base."""
    r = NORMALISE[raw].copy()
    n = r == ord("N")
    r[n] = ACGT[rng.integers(0, 4, int(n.sum()))]
    return r


def decorate(rng, r, raw, kind):
    """raw: the reference bytes the read was taken from, position by position (None on the reverse strand or past the fragment)."""
    r = r.copy()
    L = len(r)
    if kind == "lower":
        r = np.where((r >= 65) & (r <= 90), r + 32, r).astype(np.uint8)
    elif kind == "lower_runs":
        for _ in range(int(rng.integers(1, 4))):
            ln = int(rng.integers(5, 41))
            st = int(rng.integers(0, max(1, L - ln)))
            seg = r[st:st + ln]
            r[st:st + ln] = np.where((seg >= 65) & (seg <= 90), seg + 32, seg)
    elif kind in ("lower_n", "dot", "iupac"):
        pos = rng.integers(0, L, int(rng.integers(1, 4)))
        r[pos] = ord("n") if kind == "lower_n" else ord(".") if kind == "dot" else IUPAC[rng.integers(0, len(IUPAC), len(pos))]
    elif kind == "high" and raw is not None:
        n = min(L, len(raw))
        hi = raw[:n] >= 0x80
        r[:n][hi] = raw[:n][hi] - 32
    return r


def make_pairs(rng, seqs, n_pairs, read_len, frag_min, frag_max, short_frac=0.0, chimeric_frac=0.0):
    out = []
    for _ in range(n_pairs):
        si = int(rng.integers(0, len(seqs)))
        s = seqs[si]
        fl = int(rng.integers(30, read_len)) if rng.random() < short_frac else int(rng.integers(frag_min, frag_max + 1))
        st = int(rng.integers(50, len(s) - 50 - max(fl, read_len + 8)))
        raw = s[st:st + fl]
        frag = sequenced(rng, raw)
        fwd, rev = frag, COMP[frag[::-1]]
        raw_f, raw_r = raw, None
        if rng.random() < 0.5:
            fwd, rev, raw_f, raw_r = rev, fwd, None, raw
        e1 = np.concatenate([fwd, ADAPTER1])[:read_len]
        e2 = np.concatenate([rev, ADAPTER2])[:read_len]
        if chimeric_frac > 0 and rng.random() < chimeric_frac:   # ligation junction: the tail of read 1 from another locus
            j = int(rng.integers(30, read_len - 30))
            sj = seqs[int(rng.integers(0, len(seqs)))]
            pj = int(rng.integers(50, len(sj) - 50 - read_len))
            other = sj[pj:pj + read_len - j]
            tail = sequenced(rng, other)
            if rng.random() < 0.5:
                tail, other = COMP[tail[::-1]], None
            e1 = np.concatenate([e1[:j], tail])
            raw_f = None if raw_f is None and other is None else np.concatenate([raw_f[:j] if raw_f is not None else np.zeros(j, np.uint8),
                                                                               other if other is not None else np.zeros(len(tail), np.uint8)])
        k1, k2 = rng.integers(0, len(DECORATIONS), 2)
        r1 = decorate(rng, mutate(rng, e1)[:read_len], raw_f, DECORATIONS[k1])
        r2 = decorate(rng, mutate(rng, e2)[:read_len], raw_r, DECORATIONS[k2])
        out.append((r1, r2))
    return out


def write_fasta(path, seqs, names):
    with open(path, "wb") as f:
        for nm, s in zip(names, seqs):
            f.write(b">" + nm.encode() + b"\n")
            b = s.tobytes()
            for j in range(0, len(b), 80):
                f.write(b[j:j + 80] + b"\n")


def write_fastq(path, reads, prefix, suffix):
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b"@%s.%d/%s\n" % (prefix.encode(), i, suffix.encode()) + r.tobytes() + b"\n+\n" + b"I" * len(r) + b"\n")


SETS = {   # name -> (pairs, read length, fragment min, max, share of fragments shorter than the reads, chimeric share)
    "pe100": (4000, 100, 120, 500, 0.3, 0.0),
    "hic150": (2000, 150, 200, 600, 0.0, 0.5),
    "pe250": (1200, 250, 260, 700, 0.0, 0.0),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--seed", type=int, default=31)
    ap.add_argument("--normalise", choices=("none", "reads", "ref", "both"), default="none")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    rng = np.random.default_rng(a.seed)
    seqs = make_reference(rng)
    sets = {name: make_pairs(np.random.default_rng([a.seed, i]), seqs, *args) for i, (name, args) in enumerate(SETS.items())}
    norm_ref, norm_reads = a.normalise in ("ref", "both"), a.normalise in ("reads", "both")
    write_fasta(os.path.join(a.out, "ref.fa"), [NORMALISE[s] if norm_ref else s for s in seqs], ["chr1", "chr2", "chr3"])
    for name, pairs in sets.items():
        for m in (0, 1):
            write_fastq(os.path.join(a.out, "%s_%d.fq" % (name, m + 1)), [NORMALISE[p[m]] if norm_reads else p[m] for p in pairs], name, str(m + 1))


if __name__ == "__main__":
    main()
