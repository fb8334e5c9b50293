"""Inputs of tests/golden/synth_bulk_dedup (bulk-level duplicate removal of barcoded reads) on the synth_sc reference and
whitelist.  Deterministic for a seed.

Designed fragments ("sites") are repeated under several whitelisted barcodes so that the bulk groups hold entries of 1, 2, 3
and 5 records, entries tied on weight with different abundances and tied on both, barcodes one substitution away from the
whitelist (corrected into a group), reads with substitutions that lower their MAPQ (at fragments where they do), 300 copies of
one fragment (num_dups saturates at 255) and, for single-end runs, one barcode that comes back after another at one start
with a shorter read 1.  The fragment with mixed MAPQ on chr3 at 248171 is the last of the run.  Filler pairs at random
positions (never past chr3:245000) set the barcode abundances.

usage: python tools/gen_bulk_dedup.py --out DIR [--seed 2026]"""
import argparse
import gzip
import os
import random

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SC = os.path.join(ROOT, "tests", "golden", "synth_sc")
READ_LEN = 50
COMP = str.maketrans("ACGTacgtN", "TGCAtgcaN")

# (chrom, start, fragment length) of fragments that map uniquely (MAPQ 60) on the synth_sc reference
SITES = {
    "cap": ("chr1", 156357, 339),       # entries of 1, 2, 3 and 5 records
    "abund": ("chr1", 167424, 238),     # two entries of 2: the later barcode is the more abundant
    "tie": ("chr1", 199765, 210),       # two entries of 2, equally abundant
    "corr": ("chr2", 191873, 347),      # an entry made of 2 by a corrected barcode beats a more abundant single
    "single": ("chr2", 26547, 209),     # three single records
    "sat": ("chr1", 130730, 255),       # 300 records
    "lowmq": ("chr3", 246882, 221),     # the best entry's reads carry 3 substitutions (MAPQ 15), a single is clean
    "mixed": ("chr2", 129938, 234),     # one entry of a substituted (MAPQ 19) and a clean read
    "return": ("chr3", 204747, 216),    # single-end: barcode T (45-base read 1) x2, U x1, T (50 bases) x1
    "last": ("chr3", 248171, 203),      # the last group: best entry substituted (MAPQ 22), a clean single
}
MUT = {"lowmq": (3, 1), "mixed": (3, 1), "last": (3, 0)}  # (substitutions, pattern seed) of read 1


def read_ref():
    ref, name = {}, None
    for l in gzip.open(os.path.join(SC, "ref.fa.gz"), "rt"):
        l = l.strip()
        if l.startswith(">"):
            name = l[1:].split()[0]
            ref[name] = []
        else:
            ref[name].append(l)
    return {k: "".join(v).upper() for k, v in ref.items()}


def mutate(s, nm, seed):  # nm substitutions inside bases 8..41 of read 1
    a = list(s)
    for q in random.Random(seed).sample(range(8, 42), nm):
        a[q] = {"A": "C", "C": "G", "G": "T", "T": "A"}.get(a[q], "A")
    return "".join(a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--seed", type=int, default=2026)
    a = ap.parse_args()
    rng = random.Random(a.seed)
    ref = read_ref()
    wl = [l.strip() for l in open(os.path.join(SC, "whitelist.txt")) if l.strip()]
    wl_set = set(wl)
    pool = rng.sample(wl, 520)
    named, filler_pool = pool[:120], pool[120:]
    it = iter(named)
    bc = {k: next(it) for k in "ABCDEFGHIJKLMNOPQRSTU"}
    for x, y in (("E", "F"), ("G", "H")):  # E before F, G before H in the reference's order (2 bits per base, A < C < G < T)
        if bc[x] > bc[y]:
            bc[x], bc[y] = bc[y], bc[x]

    def one_off(b):  # a substitution whose only whitelisted neighbour at distance 1 is b
        for _ in range(1000):
            p, c = rng.randrange(len(b)), rng.choice("ACGT")
            m = b[:p] + c + b[p + 1:]
            if m in wl_set:
                continue
            nb = {m[:q] + d + m[q + 1:] for q in range(len(m)) for d in "ACGT"} & wl_set
            if nb == {b}:
                return m
        raise RuntimeError("no barcode one substitution away from " + b)

    pairs = []  # (chrom, start, length, barcode, substitutions, seed, read-1 length)

    def site(key, b, n, mut=False, r1_len=READ_LEN):
        c, p, L = SITES[key]
        nm, seed = MUT[key] if mut else (0, 0)
        pairs.extend((c, p, L, b, nm, seed, r1_len) for _ in range(n))

    site("cap", bc["A"], 1); site("cap", bc["B"], 2); site("cap", bc["C"], 3); site("cap", bc["D"], 5)
    site("abund", bc["E"], 2); site("abund", bc["F"], 2)
    site("tie", bc["G"], 2); site("tie", bc["H"], 2)
    site("corr", bc["I"], 1); site("corr", one_off(bc["I"]), 1); site("corr", bc["J"], 1)
    site("single", bc["K"], 1); site("single", bc["L"], 1); site("single", bc["M"], 1)
    for b in named[21:81]:
        site("sat", b, 5)
    site("lowmq", bc["N"], 2, mut=True); site("lowmq", bc["O"], 1)
    site("mixed", bc["P"], 1, mut=True); site("mixed", bc["P"], 1); site("mixed", bc["Q"], 1)
    site("return", bc["T"], 2, r1_len=45); site("return", bc["U"], 1, r1_len=45); site("return", bc["T"], 1)
    site("last", bc["R"], 2, mut=True); site("last", bc["S"], 1)
    # abundances: filler copies of the named barcodes, then 3000 pairs over the rest of the pool
    extra = dict(A=40, B=30, C=10, D=5, E=8, F=20, G=15, H=15, I=3, J=25, K=7, L=12, M=9, N=30, O=4, P=6, Q=11, R=35, S=5, T=30, U=10)
    fill = [bc[k] for k, n in extra.items() for _ in range(n)] + [rng.choice(filler_pool) for _ in range(3000)]
    lens = {c: len(s) for c, s in ref.items()}
    for b in fill:
        c = rng.choice(sorted(lens))
        L = rng.randrange(180, 400)
        p = rng.randrange(1000, (245000 if c == "chr3" else lens[c]) - 1000)
        pairs.append((c, p, L, b, 0, 0, READ_LEN))
    rng.shuffle(pairs)
    os.makedirs(a.out, exist_ok=True)
    with gzip.GzipFile(os.path.join(a.out, "read1.fq.gz"), "wb", mtime=0) as f1, \
            gzip.GzipFile(os.path.join(a.out, "read2.fq.gz"), "wb", mtime=0) as f2, \
            gzip.GzipFile(os.path.join(a.out, "barcode.fq.gz"), "wb", mtime=0) as fb:
        for i, (c, p, L, b, nm, seed, r1_len) in enumerate(pairs):
            s = ref[c][p:p + L]
            r1 = mutate(s[:READ_LEN], nm, seed)[:r1_len]
            r2 = s[L - READ_LEN:].translate(COMP)[::-1]
            f1.write(b"@bd.%d/1\n%s\n+\n%s\n" % (i, r1.encode(), b"I" * len(r1)))
            f2.write(b"@bd.%d/2\n%s\n+\n%s\n" % (i, r2.encode(), b"I" * len(r2)))
            fb.write(b"@bd.%d\n%s\n+\n%s\n" % (i, b.encode(), b"I" * len(b)))


if __name__ == "__main__":
    main()
