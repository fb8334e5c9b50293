"""Seeded synthetic inputs for the runs that cross reference-batch, taskloop-chunk, lane and CLI-call boundaries
(test_gpu_batch_boundaries, test_gpu_cli_runs): a 4.5 Mbp reference with planted repeats, read pairs, cell barcodes against a
whitelist, and FASTQ text, made with vectorised numpy.

The share of pairs that reach the last overflow tier is kept small on purpose.  That tier reserves about 3.4 MB of scratch
per pair (65,536 hits, 8,192 candidates and 8,192 draft mappings per read, DESIGN §3), sized for the fraction of pairs a
genome sends there (0.13 % of the benchmark's pairs; 1 % reach tier 1, about 75 KB each).  So the repeat family stays below
the tier-1 candidate capacity, 5 % of the fragments come from the planted segments, and reads longer than twice
`max_read_length` are 0.5 % of the mates."""
import functools

import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.full(256, ord("N"), dtype=np.uint8)
COMP[list(b"ACGTN")] = list(b"TGCAN")
N_SEQ, SEQ_LEN = 3, 1_500_000
SEG_LEN, SEG_COPIES = 3000, 12


@functools.lru_cache(maxsize=1)
def reference():
    """(sequences, segment copy starts as (rid, pos)): random bases, per sequence one 3 kb segment in 12 exact copies, a
    300 bp family in 60 copies over the reference (0.5 % diverged), short N runs."""
    rng = np.random.default_rng(20261018)
    seqs, copies = [], []
    fam = rng.integers(0, 4, 300)
    for s in range(N_SEQ):
        a = rng.integers(0, 4, SEQ_LEN)
        seg = rng.integers(0, 4, SEG_LEN)
        st = np.sort(rng.choice(SEQ_LEN // SEG_LEN - 1, SEG_COPIES, replace=False)) * SEG_LEN
        for p in st:
            a[p:p + SEG_LEN] = seg
            copies.append((s, int(p)))
        for p in rng.integers(0, SEQ_LEN - 300, 20):
            f = fam.copy()
            m = rng.random(300) < 0.005
            f[m] = rng.integers(0, 4, int(m.sum()))
            a[p:p + 300] = f
        a = ACGT[a]
        for p in rng.integers(0, SEQ_LEN - 50, 20):
            a[p:p + int(rng.integers(1, 50))] = ord("N")
        seqs.append(a)
    return seqs, np.array(copies)


def _ragged(rows, lens):
    """Concatenation of rows[i, :lens[i]] and its uint32 offsets."""
    keep = np.arange(rows.shape[1])[None, :] < lens[:, None]
    off = np.zeros(len(lens) + 1, dtype=np.uint32)
    off[1:] = np.cumsum(lens)
    return np.ascontiguousarray(rows[keep]), off


def make_reads(n, seed, hic=False, length=None, in_segment=()):
    """n pairs: (seq1, off1, seq2, off2).  5 % of the fragments lie inside a planted segment copy (twelve equally good
    pairs; these reads overflow to tier 1).  Mates are `length` bases long if given, else 50 (95.5 %), 100 (4 %) or 150
    (0.5 %).  The pairs listed in `in_segment` always come from a segment copy and are never junk.  For Hi-C (`hic`) a
    third of the mates are chimeric: the tail from another locus.  1 % substitutions, a few Ns, 1 % junk pairs.  Made in
    pieces of 65,536 pairs to bound the index arrays."""
    force = np.asarray(in_segment, dtype=np.int64)
    parts = [_read_piece(min(65536, n - p0), seed * 1000 + p0 // 65536, hic, length, force[(force >= p0) & (force < p0 + 65536)] - p0)
             for p0 in range(0, n, 65536)]
    r1, l1, r2, l2 = (np.concatenate([p[i] for p in parts]) for i in range(4))
    s1, o1 = _ragged(r1, l1)
    s2, o2 = _ragged(r2, l2)
    return s1, o1, s2, o2


def _read_piece(n, seed, hic, length, force):
    seqs, copies = reference()
    ref = np.concatenate(seqs)
    rng = np.random.default_rng(seed)
    L = length or 150
    l1, l2 = (np.full(n, L) if length else rng.choice([50, 100, 150], n, p=[0.955, 0.04, 0.005]) for _ in range(2))
    fl = rng.integers(np.maximum(l1, l2) + 20, 501)
    rid = rng.integers(0, N_SEQ, n)
    st = rng.integers(0, SEQ_LEN - 600, n)
    inseg = rng.random(n) < 0.05
    inseg[force] = True
    c = copies[rng.integers(0, len(copies), int(inseg.sum()))]
    fl[inseg] = np.minimum(fl[inseg], SEG_LEN - 10)
    rid[inseg] = c[:, 0]
    st[inseg] = c[:, 1] + rng.integers(0, SEG_LEN - fl[inseg] + 1)
    base = rid * SEQ_LEN + st
    ar = np.arange(L)[None, :]
    left = ref[base[:, None] + ar]
    right = COMP[ref[(base + fl - 1)[:, None] - ar]]
    fwd = (rng.random(n) < 0.5)[:, None]
    r1, r2 = np.where(fwd, left, right), np.where(fwd, right, left)
    if hic:
        for r in (r1, r2):
            chim = np.flatnonzero(rng.random(n) < 0.33)
            cut = rng.integers(40, L - 39, len(chim))
            other = rng.integers(0, N_SEQ, len(chim)) * SEQ_LEN + rng.integers(0, SEQ_LEN - L, len(chim))
            r[chim] = np.where(ar < cut[:, None], r[chim], ref[other[:, None] + ar])
    for r in (r1, r2):
        m = rng.random(r.shape) < 0.01
        r[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
        r[rng.random(r.shape) < 0.0005] = ord("N")
    junk = rng.random(n) < 0.01
    junk[force] = False
    r1[junk] = ACGT[rng.integers(0, 4, (int(junk.sum()), L))]
    return r1, l1, r2, l2


def make_barcodes(n, seed, path, bc_len=16):
    """A 3,000-entry whitelist written to `path` and n barcodes (bases, qualities) from 800 of its cells: 8 % with one
    substitution, 4 % with two, 3 % with an N, 3 % random; Phred qualities 0 to 41."""
    rng = np.random.default_rng(seed)
    wl = ACGT[rng.integers(0, 4, (3000, bc_len))]
    with open(path, "wb") as f:
        f.write(b"".join(bytes(r) + b"\n" for r in wl))
    obs = wl[rng.integers(0, 800, n)]
    kind = rng.random(n)
    for k, (lo, hi) in enumerate(((0.0, 0.08), (0.08, 0.12))):
        rows = np.flatnonzero((kind >= lo) & (kind < hi))
        for j in range(k + 1):
            pos = rng.integers(0, bc_len, len(rows)) if j == 0 else (pos + rng.integers(1, bc_len, len(rows))) % bc_len
            cur = np.searchsorted(ACGT, obs[rows, pos])
            obs[rows, pos] = ACGT[(cur + rng.integers(1, 4, len(rows))) % 4]
    rows = np.flatnonzero((kind >= 0.12) & (kind < 0.15))
    obs[rows, rng.integers(0, bc_len, len(rows))] = ord("N")
    rows = np.flatnonzero((kind >= 0.15) & (kind < 0.18))
    obs[rows] = ACGT[rng.integers(0, 4, (len(rows), bc_len))]
    quals = (rng.integers(0, 42, (n, bc_len)) + 33).astype(np.uint8)
    return np.ascontiguousarray(obs.reshape(-1)), np.ascontiguousarray(quals.reshape(-1)), bc_len


def fastq(seqs, length, prefix=b"r"):
    """4-line FASTQ text of equal-length reads (a uint8 concatenation): names prefix + 8-digit index, qualities 'I'."""
    n = len(seqs) // length
    digits = (np.arange(n, dtype=np.int64)[:, None] // 10 ** np.arange(7, -1, -1)[None, :]) % 10 + ord("0")
    head = np.frombuffer(b"@" + prefix, dtype=np.uint8)
    cols = [np.broadcast_to(head, (n, len(head))), digits.astype(np.uint8), np.full((n, 1), ord("\n"), np.uint8),
            seqs.reshape(n, length), np.broadcast_to(np.frombuffer(b"\n+\n", np.uint8), (n, 3)),
            np.full((n, length), ord("I"), np.uint8), np.full((n, 1), ord("\n"), np.uint8)]
    return np.concatenate(cols, axis=1).tobytes()
