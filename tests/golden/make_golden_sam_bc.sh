#!/bin/bash
# Regenerates tests/golden/synth_sam_bc/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# --SAM with cell barcodes on the synth_sc inputs (and synth_bc_error2's barcodes and dense whitelist at --bc-error-threshold 2,
# synth_barcode_translate's tables).  The identity case is compared with cmp; the reference's exit status and message for a
# barcode missing from the translation table are asserted.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
REF=$(cd ../.. && pwd)/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
BE=$GOLDEN/synth_bc_error2
TR=$GOLDEN/synth_barcode_translate
RF=$GOLDEN/synth_read_format
rm -rf synth_sam_bc && mkdir -p synth_sam_bc
cd synth_sam_bc
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
for f in ref.fa read1.fq read2.fq barcode.fq; do gzip -dc $SC/$f.gz > $TMP/$f; done
gzip -dc $BE/barcode.fq.gz > $TMP/barcode_e2.fq
gzip -dc $RF/bc24.fq.gz > $TMP/bc24.fq
$REF -i -r $TMP/ref.fa -o $TMP/ref.index 2> /dev/null
WL="--barcode-whitelist $SC/whitelist.txt"
PE="-1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/barcode.fq"
SE="-1 $TMP/read1.fq -b $TMP/barcode.fq"
sc() { name=$1; shift; $REF -x $TMP/ref.index -r $TMP/ref.fa -t 1 --SAM "$@" -o $name 2> /dev/null; }
sc pe_atac.sam --preset atac $WL $PE
sc se_atac.sam --preset atac $WL $SE
sc pe_q0dedup.sam -q 0 --remove-pcr-duplicates $WL $PE
sc se_q0dedup.sam -q 0 --remove-pcr-duplicates $WL $SE
sc pe_nowl.sam --preset atac $PE
sc pe_notinwl.sam --preset atac $WL --output-mappings-not-in-whitelist $PE
sc pe_n3q0.sam -n 3 -q 0 $WL $PE
sc pe_bcerr2.sam --preset atac --bc-error-threshold 2 --barcode-whitelist $BE/dense.txt.gz -1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/barcode_e2.fq
sc pe_rc16.sam --preset atac $WL $PE --barcode-translate $TR/rc16.txt.gz
sc pe_half8.sam --preset atac $WL $PE --barcode-translate $TR/half8.txt.gz
# identity case: the barcode inside a longer read gives the same file
sc $TMP/o.sam --preset atac $WL -1 $TMP/read1.fq -2 $TMP/read2.fq -b $TMP/bc24.fq --read-format bc:8:23
cmp pe_atac.sam $TMP/o.sam
# a table without one of the output barcodes: the reference stops with status 255 and its message
set +e
$REF --SAM --preset atac $WL $PE --barcode-translate $TR/missing_rc16.txt.gz -x $TMP/ref.index -r $TMP/ref.fa -t 1 -o $TMP/o.sam 2> $TMP/err.txt
status=$?
set -e
test $status -eq 255
grep -qx "Barcode does not exist in the translation table." $TMP/err.txt
md5sum *.sam > md5.txt
gzip -9 -n *.sam
