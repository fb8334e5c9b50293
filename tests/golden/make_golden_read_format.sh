#!/bin/bash
# Regenerates tests/golden/synth_read_format/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by
# oracle/Makefile): --read-format cases.  The inputs are derived from synth_sc / synth_small / synth_hic without randomness
# and committed.  Identity cases: a derived input with its format must give an existing golden, which the reference's own
# output is compared against (cmp).  New outputs are committed.  Reads the other golden directories and leaves them alone.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
REF=$(cd ../.. && pwd)/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
SMALL=$GOLDEN/synth_small
HIC=$GOLDEN/synth_hic
rm -rf synth_read_format && mkdir -p synth_read_format
cd synth_read_format
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
for d in sc small hic; do mkdir -p $TMP/$d; done
for f in ref.fa read1.fq read2.fq barcode.fq; do gzip -dc $SC/$f.gz > $TMP/sc/$f; done
for f in ref.fa read1.fq read2.fq; do gzip -dc $SMALL/$f.gz > $TMP/small/$f; gzip -dc $HIC/$f.gz > $TMP/hic/$f; done
# derived inputs (4-line FASTQ; bases are upper-case ACGTN, so a reverse complement taken twice is the identity)
python3 - "$TMP" <<'EOF'
import sys
tmp = sys.argv[1]
def records(path):
    lines = open(path).read().split("\n")
    return [lines[i:i + 4] for i in range(0, len(lines) - 3, 4)]
def write(path, recs):
    open(path, "w").write("".join("%s\n%s\n%s\n%s\n" % tuple(r) for r in recs))
rc = lambda s: s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]
bc = records(tmp + "/sc/barcode.fq")
# barcode at 8..23 of a 24-base read (bc:8:23)
write("bc24.fq", [[h, "GATTACAC" + s, p, "FFFFFFFF" + q] for h, s, p, q in bc])
# barcode sequenced on the other strand (bc:0:15:-)
write("bc_rc.fq", [[h, rc(s), p, q[::-1]] for h, s, p, q in bc])
# barcode in two segments with 4 filler bases between them (bc:0:7,bc:12:19)
write("bc_split.fq", [[h, s[:8] + "TTTT" + s[8:], p, q[:8] + "####" + q[8:]] for h, s, p, q in bc])
# barcode (with its qualities) in front of read 1 (-1 and -b the same file: bc:0:15,r1:16:-1)
write("r1_bc.fq", [[h, b[1] + s, p, b[3] + q] for (h, s, p, q), b in zip(records(tmp + "/sc/read1.fq"), bc)])
# read 2 of synth_small on the other strand (r2:0:-1:-)
write("small_read2_rc.fq", [[h, rc(s), p, q[::-1]] for h, s, p, q in records(tmp + "/small/read2.fq")])
EOF
$REF -i -r $TMP/sc/ref.fa -o $TMP/sc/ref.index 2> /dev/null
$REF -i -r $TMP/small/ref.fa -o $TMP/small/ref.index 2> /dev/null
$REF -i -r $TMP/hic/ref.fa -o $TMP/hic/ref.index 2> /dev/null
sc() { $REF --preset atac -x $TMP/sc/ref.index -r $TMP/sc/ref.fa --barcode-whitelist $SC/whitelist.txt -t 1 "$@" 2> /dev/null; }
same() { gzip -dc $1 | cmp - $2; }
# identity cases
sc -1 $TMP/sc/read1.fq -2 $TMP/sc/read2.fq -b bc24.fq --read-format bc:8:23 -o $TMP/o.bed; same $SC/sc_whitelist.bed.gz $TMP/o.bed
sc -1 $TMP/sc/read1.fq -b bc24.fq --read-format bc:8:23 -o $TMP/o.bed; same $SC/se_sc_whitelist.bed.gz $TMP/o.bed
sc -1 $TMP/sc/read1.fq -2 $TMP/sc/read2.fq -b bc_rc.fq --read-format bc:0:15:- -o $TMP/o.bed; same $SC/sc_whitelist.bed.gz $TMP/o.bed
sc -1 $TMP/sc/read1.fq -2 $TMP/sc/read2.fq -b bc_split.fq --read-format bc:0:7,bc:12:19 -o $TMP/o.bed; same $SC/sc_whitelist.bed.gz $TMP/o.bed
sc -1 r1_bc.fq -2 $TMP/sc/read2.fq -b r1_bc.fq --read-format bc:0:15,r1:16:-1 -o $TMP/o.bed; same $SC/sc_whitelist.bed.gz $TMP/o.bed
$REF --preset chip --read-format r2:0:-1:- -x $TMP/small/ref.index -r $TMP/small/ref.fa -1 $TMP/small/read1.fq -2 small_read2_rc.fq -o $TMP/o.bed -t 1 2> /dev/null
same $SMALL/chip.bed.gz $TMP/o.bed
# new outputs
small() { name=$1; shift; $REF "$@" -x $TMP/small/ref.index -r $TMP/small/ref.fa -o $name -t 1 2> /dev/null; }
small pe_chip_r1_0_39_r2_5.bed --preset chip --read-format r1:0:39,r2:5:-1 -1 $TMP/small/read1.fq -2 $TMP/small/read2.fq
small se_r1_10.bed --read-format r1:10:-1 -1 $TMP/small/read1.fq
small pe_chip_rev.sam --preset chip --SAM --read-format r1:2:46:-,r2:0:44:- -1 $TMP/small/read1.fq -2 $TMP/small/read2.fq
$REF --preset hic --read-format r1:0:99,r2:20:-1 -x $TMP/hic/ref.index -r $TMP/hic/ref.fa -1 $TMP/hic/read1.fq -2 $TMP/hic/read2.fq -o hic_r1_0_99_r2_20.pairs -t 1 2> /dev/null
md5sum *.bed *.sam *.pairs > md5.txt
gzip -9 -n *.fq *.bed *.sam *.pairs
