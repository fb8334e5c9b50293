#!/bin/bash
# Regenerates tests/golden/synth_bytes/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# reads and a reference beyond upper-case ACGTN (tools/gen_bytes.py: soft-masking, IUPAC codes, bytes 0x80-0xFF in the
# reference; lower case, 'n', '.', IUPAC codes and bytes 0x60-0xDF in the reads).  2x100 pairs for BED / TagAlign / PAF / SAM,
# their read 1 for single-end, 2x150 for --preset hic, 2x250 for a grown context.  Outputs are committed.
# stats.txt: for each output, the number of lines that differ (multiset difference, both ways) from the same run on normalised
# inputs (gen_bytes.py --normalise): reads normalised, reference normalised, both.
set -e
cd "$(dirname "$0")"
REPO=$(cd ../.. && pwd)
REF=$REPO/oracle/_ref/chromap
rm -rf synth_bytes && mkdir -p synth_bytes
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
python $REPO/tools/gen_bytes.py --out synth_bytes
for n in reads ref both; do python $REPO/tools/gen_bytes.py --out $TMP/$n --normalise $n; done
# name|options|reads (chromap's -1 / -2 files, without the _1.fq / _2.fq)|single-end
CASES="chip.bed|--preset chip|pe100|
q0.bed|-q 0|pe100|
atac.bed|--preset atac|pe100|
chip.tagalign|--preset chip --TagAlign|pe100|
q0.paf|--PAF -q 0|pe100|
pe_q0.sam|--SAM -q 0|pe100|
se_q0.sam|--SAM -q 0|pe100|se
se_q0.bed|-q 0|pe100|se
hic.pairs|--preset hic|hic150|
hic_q0.pairs|--preset hic -q 0|hic150|
pe250_chip.bed|--preset chip|pe250|
pe250_q0.sam|--SAM -q 0|pe250|
rf_rev.bed|--preset chip --read-format r1:0:-1:-,r2:0:-1:-|pe100|"
run() {   # dir name options reads se
  local d=$1 name=$2 opts=$3 reads=$4 se=$5
  local r2="-2 $d/${reads}_2.fq"
  [ -n "$se" ] && r2=""
  $REF $opts -x $d/ref.index -r $d/ref.fa -1 $d/${reads}_1.fq $r2 -o $d/$name -t 1 2> /dev/null
}
for d in synth_bytes $TMP/reads $TMP/ref $TMP/both; do $REF -i -r $d/ref.fa -o $d/ref.index 2> /dev/null; done
: > synth_bytes/stats.txt
while IFS='|' read -r name opts reads se; do
  counts=""
  for d in synth_bytes $TMP/reads $TMP/ref $TMP/both; do run $d "$name" "$opts" $reads "$se"; done
  for n in reads ref both; do
    counts="$counts $(python3 -c 'import collections, sys
a, b = (collections.Counter(open(p, "rb").read().splitlines()) for p in sys.argv[1:3])
print(sum(((a - b) + (b - a)).values()))' synth_bytes/$name $TMP/$n/$name)"
  done
  echo "$name$counts" >> synth_bytes/stats.txt
done <<< "$CASES"
cd synth_bytes
rm -f ref.index
md5sum *.bed *.tagalign *.paf *.sam *.pairs > md5.txt
gzip -9 -n ref.fa *.fq *.bed *.tagalign *.paf *.sam *.pairs
