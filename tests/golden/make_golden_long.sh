#!/bin/bash
# Regenerates tests/golden/synth_long/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# reads longer than 160 bases (tests/long_reads_inputs.py, seeded) on synth_sc's reference, every output format the GPU path
# writes, one thread.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
ROOT=$(cd ../.. && pwd)
REF=$ROOT/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
rm -rf synth_long && mkdir -p synth_long
cd synth_long
(cd "$ROOT" && python3 -m tests.long_reads_inputs "$GOLDEN/synth_long")
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
gzip -dc $SC/ref.fa.gz > $TMP/ref.fa
$REF -i -r $TMP/ref.fa -o $TMP/ref.index 2> /dev/null
run() { name=$1; shift; $REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 "$@" -o $name 2> /dev/null; }
pe() { echo "-1 pe$1_1.fq.gz -2 pe$1_2.fq.gz"; }
run pe250_chip.bed --preset chip $(pe 250)
run pe300_chip.bed --preset chip $(pe 300)
run mixed_chip.bed --preset chip -1 mixed_1.fq.gz -2 mixed_2.fq.gz
run se250_chip.bed --preset chip -1 se250_1.fq.gz
run pe250_atac.bed --preset atac $(pe 250)
run pe300_atac.bed --preset atac $(pe 300)
run pe250_chip.tagalign --preset chip --TagAlign $(pe 250)
run pe250_q0.sam -q 0 --SAM $(pe 250)
run mixed_q0.sam -q 0 --SAM -1 mixed_1.fq.gz -2 mixed_2.fq.gz
run se250_q0.sam -q 0 --SAM -1 se250_1.fq.gz
run pe250_sc_atac.bed --preset atac $(pe 250) -b barcode.fq.gz --barcode-whitelist $SC/whitelist.txt
run hic250.pairs --preset hic -1 hic250_1.fq.gz -2 hic250_2.fq.gz
md5sum *.bed *.tagalign *.sam *.pairs > md5.txt
gzip -9 -n *.bed *.tagalign *.sam *.pairs
