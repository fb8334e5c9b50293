#!/bin/bash
# Regenerates tests/golden/synth_edges/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# a reference of one 60 kbp sequence and 50 short ones (20 bp .. 3 kbp), with 70% of the fragments starting or ending within
# 40 bp of a sequence's ends.  2x50 reads for the BED and SAM outputs, 2x150 (hic_read*.fq) for --preset hic.  Outputs are committed.
set -e
cd "$(dirname "$0")"
REPO=$(cd ../.. && pwd)
REF=$REPO/oracle/_ref/chromap
EDGES="--seed 21 --n-seq 1 --seq-len 60000 --short-seqs 50 --edge-frac 0.7 --repeat-copies 0 --fam-copies 150"
rm -rf synth_edges && mkdir -p synth_edges
python $REPO/tools/gen_synth.py --out synth_edges $EDGES --n-pairs 3000 --read-len 50
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
python $REPO/tools/gen_synth.py --out $TMP $EDGES --n-pairs 1500 --read-len 150 --chimeric-frac 0.3
cd synth_edges
cmp ref.fa $TMP/ref.fa
mv $TMP/read1.fq hic_read1.fq; mv $TMP/read2.fq hic_read2.fq
$REF -i -r ref.fa -o ref.index 2> /dev/null
run() { name=$1; shift; $REF "$@" -x ref.index -r ref.fa -1 read1.fq -2 read2.fq -o $name -t 1 2> /dev/null; }
runse() { name=$1; shift; $REF "$@" -x ref.index -r ref.fa -1 read1.fq -o $name -t 1 2> /dev/null; }
run chip.bed --preset chip
run q0.bed -q 0
run e15q0.bed -e 15 -q 0
run e1q0.bed -e 1 -q 0
run atac.bed --preset atac
runse se_q0.bed -q 0
run pe_q0.sam --SAM -q 0
runse se_q0.sam --SAM -q 0
$REF --preset hic -q 0 -x ref.index -r ref.fa -1 hic_read1.fq -2 hic_read2.fq -o hic_q0.pairs -t 1 2> /dev/null
md5sum *.bed *.sam *.pairs > md5.txt
gzip -9 -n ref.fa read1.fq read2.fq hic_read1.fq hic_read2.fq *.bed *.sam *.pairs
rm -f ref.index
