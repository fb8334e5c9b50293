#!/bin/bash
# Regenerates tests/golden/synth_params/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# the synth_small reads mapped at other index shapes (k, w) and other mapping knobs (-e, -n, -s, -f, --drop-repetitive-reads,
# --min-read-length).  Reads synth_small/ and leaves it alone.  Outputs are committed.
set -e
cd "$(dirname "$0")"
REPO=$(cd ../.. && pwd)
REF=$REPO/oracle/_ref/chromap
IN=$(pwd)/synth_small
rm -rf synth_params && mkdir -p synth_params
cd synth_params
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
gzip -dc $IN/ref.fa.gz > $TMP/ref.fa
gzip -dc $IN/read1.fq.gz > $TMP/read1.fq
gzip -dc $IN/read2.fq.gz > $TMP/read2.fq
# one index per shape; --min-frag-length picks (19, 10) up to 80 and (23, 11) above (chromap_driver.cc:277-289)
$REF -i -r $TMP/ref.fa -o $TMP/k17w7.index 2> /dev/null
$REF -i --min-frag-length 70 -r $TMP/ref.fa -o $TMP/k19w10.index 2> /dev/null
$REF -i --min-frag-length 100 -r $TMP/ref.fa -o $TMP/k23w11.index 2> /dev/null
$REF -i -k 28 -w 20 -r $TMP/ref.fa -o $TMP/k28w20.index 2> /dev/null
$REF -i -k 16 -w 5 -r $TMP/ref.fa -o $TMP/k16w5.index 2> /dev/null
run() { name=$1; ix=$2; shift 2; $REF "$@" -x $TMP/$ix.index -r $TMP/ref.fa -1 $TMP/read1.fq -2 $TMP/read2.fq -o $name.bed -t 1 2> /dev/null; }
runse() { name=$1; ix=$2; shift 2; $REF "$@" -x $TMP/$ix.index -r $TMP/ref.fa -1 $TMP/read1.fq -o $name.bed -t 1 2> /dev/null; }
run mfl70 k19w10
run mfl70_e15 k19w10 -e 15
run mfl100_q0 k23w11 -q 0
run mfl100_chip k23w11 --preset chip
runse mfl100_se_q0 k23w11 -q 0
run k28w20 k28w20
run k16w5_q0 k16w5 -q 0
run e15q0 k17w7 -e 15 -q 0
run e7q0 k17w7 -e 7 -q 0
run e1q0 k17w7 -e 1 -q 0
run n8q0 k17w7 -n 8 -q 0
run s1q0 k17w7 -s 1 -q 0
run s4 k17w7 -s 4
run f20_200q0 k17w7 -f 20,200 -q 0
run drop30q0 k17w7 --drop-repetitive-reads 30 -q 0
run minlen45q0 k17w7 --min-read-length 45 -q 0
runse se_e15n8q0 k17w7 -e 15 -n 8 -q 0
md5sum *.bed > md5.txt
gzip -9 -n *.bed
