#!/bin/bash
# Regenerates tests/golden/synth_bc_error2/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by
# oracle/Makefile): --bc-error-threshold 2.  The inputs are derived from synth_sc by seeded Python and committed gzipped:
#   barcode.fq   synth_sc's barcodes with about 5 % two substitutions, 2 % one substitution and one N, 1 % two Ns and 1 % three Ns
#   dense.txt    synth_sc's whitelist plus an entry two substitutions away from every third entry, so that corrections at
#                distance 1 and 2 compete
# stats.txt keeps each run's "Number of barcodes in whitelist / corrected barcodes".  Identity cases are compared with cmp.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
REF=$(cd ../.. && pwd)/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
RF=$GOLDEN/synth_read_format
rm -rf synth_bc_error2 && mkdir -p synth_bc_error2
cd synth_bc_error2
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
for f in ref.fa read1.fq read2.fq barcode.fq; do gzip -dc $SC/$f.gz > $TMP/$f; done
gzip -dc $RF/bc24.fq.gz > $TMP/bc24.fq
python3 - "$TMP/barcode.fq" "$SC/whitelist.txt" <<'EOF'
import random, sys
g = random.Random(2)
lines = open(sys.argv[1]).read().split("\n")[:-1]
def change(s, pos, to=None):
    c = to or g.choice([b for b in "ACGT" if b != s[pos]])
    return s[:pos] + c + s[pos + 1:]
wl = open(sys.argv[2]).read().split()
extra = []
for w in wl[::3]:
    a, b = g.sample(range(len(w)), 2)
    extra.append(change(change(w, a), b))
seen = set(wl)
extra = [e for e in extra if not (e in seen or seen.add(e))]
open("dense.txt", "w").write("\n".join(wl + extra) + "\n")
# 4 % of the barcodes are the added entries themselves, so that they have abundances; the errors then apply to any barcode
for r in range(1, len(lines), 4):
    s, u = lines[r], g.random()
    if g.random() < 0.04: s = g.choice(extra)
    pos = g.sample(range(len(s)), 3)
    if u < 0.05: s = change(change(s, pos[0]), pos[1])
    elif u < 0.07: s = change(change(s, pos[0]), pos[1], "N")
    elif u < 0.08: s = change(change(s, pos[0], "N"), pos[1], "N")
    elif u < 0.09: s = change(change(change(s, pos[0], "N"), pos[1], "N"), pos[2], "N")
    lines[r] = s
open("barcode.fq", "w").write("\n".join(lines) + "\n")
EOF
$REF -i -r $TMP/ref.fa -o $TMP/ref.index 2> /dev/null
sc() { name=$1; shift; $REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 --bc-error-threshold 2 "$@" -o $name.bed 2> $TMP/$name.log
       echo "$name $(grep -o 'Number of barcodes in whitelist: [0-9]*' $TMP/$name.log | grep -o '[0-9]*$') $(grep -o 'Number of corrected barcodes: [0-9]*' $TMP/$name.log | grep -o '[0-9]*$')" >> stats.txt; }
PE="-1 $TMP/read1.fq -2 $TMP/read2.fq -b barcode.fq"
SE="-1 $TMP/read1.fq -b barcode.fq"
WL="--barcode-whitelist $SC/whitelist.txt"
DENSE="--barcode-whitelist dense.txt"
sc pe_wl --preset atac $WL $PE
sc pe_dense --preset atac $DENSE $PE
sc pe_dense_p04 --preset atac $DENSE --bc-probability-threshold 0.4 $PE
sc pe_dense_notinwl --preset atac $DENSE --output-mappings-not-in-whitelist $PE
sc se_dense --preset atac $DENSE $SE
sc pe_orig --preset atac $WL -1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/barcode.fq
# identity cases: without a whitelist the threshold changes nothing; a barcode cut from inside a longer read corrects the same
$REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 --bc-error-threshold 2 --preset atac -1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/barcode.fq -o $TMP/o.bed 2> /dev/null
gzip -dc $SC/sc_nowhitelist.bed.gz | cmp - $TMP/o.bed
$REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 --bc-error-threshold 2 --preset atac $WL -1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/bc24.fq --read-format bc:8:23 -o $TMP/o.bed 2> /dev/null
cmp pe_orig.bed $TMP/o.bed
md5sum *.bed > md5.txt
gzip -9 -n *.bed barcode.fq dense.txt
