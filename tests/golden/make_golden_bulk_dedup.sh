#!/bin/bash
# Regenerates tests/golden/synth_bulk_dedup/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# barcoded BED with duplicates removed at bulk level (the reference's default for single-cell data in a low-memory run) on the
# inputs of tools/gen_bulk_dedup.py (synth_sc's reference and whitelist), plus one in-memory run, where the level changes nothing.
# stats.txt keeps each run's "Number of output mappings (passed filters)" line.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
ROOT=$(cd ../.. && pwd)
REF=$ROOT/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
TR=$GOLDEN/synth_barcode_translate
rm -rf synth_bulk_dedup && mkdir -p synth_bulk_dedup
cd synth_bulk_dedup
python3 $ROOT/tools/gen_bulk_dedup.py --out . --seed 2026
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
gzip -dc $SC/ref.fa.gz > $TMP/ref.fa
for f in read1.fq read2.fq barcode.fq; do gzip -dc $f.gz > $TMP/$f; done
$REF -i -r $TMP/ref.fa -o $TMP/ref.index 2> /dev/null
WL="--barcode-whitelist $SC/whitelist.txt"
PE="-1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/barcode.fq"
SE="-1 $TMP/read1.fq -b $TMP/barcode.fq"
: > stats.txt
run() {
  name=$1; shift
  $REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 "$@" -o $name 2> $TMP/err.txt
  echo "$name $(grep 'Number of output mappings (passed filters)' $TMP/err.txt)" >> stats.txt
}
run pe_chip.bed --preset chip $WL $PE
run se_chip.bed --preset chip $WL $SE
run pe_q0.bed --low-mem --remove-pcr-duplicates -q 0 $WL $PE
run se_q0.bed --low-mem --remove-pcr-duplicates -q 0 $WL $SE
run pe_atac_bulk.bed --preset atac --remove-pcr-duplicates-at-bulk-level $WL $PE
run pe_chip_rc16.bed --preset chip $WL $PE --barcode-translate $TR/rc16.txt.gz
run pe_inmem_q0.bed --remove-pcr-duplicates -q 0 $WL $PE
md5sum *.bed > md5.txt
gzip -9 -n *.bed
