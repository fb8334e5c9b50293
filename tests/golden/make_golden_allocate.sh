#!/bin/bash
# Regenerates tests/golden/synth_allocate/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by oracle/Makefile):
# --allocate-multi-mappings with its distance and seed, on synth_small (paired-end, single-end, TagAlign) and synth_sc (barcoded
# paired-end and single-end, with the whitelist).  stats.txt keeps the four log lines of each run (mapping_processor.h:363,431-435,
# chromap.h:1348-1350), "== case" before them, the time removed.  Two more checks, by cmp and by exit status:
#   - in low-memory mode (--preset chip) the option changes nothing;
#   - with no multi-mapping at all (the first three pairs) the reference aborts on its assertion.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
REF=$(cd ../.. && pwd)/oracle/_ref/chromap
SM=$GOLDEN/synth_small
SC=$GOLDEN/synth_sc
rm -rf synth_allocate && mkdir -p synth_allocate
cd synth_allocate
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
for f in ref.fa read1.fq read2.fq; do gzip -dc $SM/$f.gz > $TMP/sm_$f; done
for f in ref.fa read1.fq read2.fq barcode.fq; do gzip -dc $SC/$f.gz > $TMP/sc_$f; done
$REF -i -r $TMP/sm_ref.fa -o $TMP/sm.index 2> /dev/null
$REF -i -r $TMP/sc_ref.fa -o $TMP/sc.index 2> /dev/null
run() { name=$1; ext=$2; d=$3; shift 3
        $REF -x $TMP/$d.index -r $TMP/${d}_ref.fa -t 1 --allocate-multi-mappings "$@" -o $name.$ext 2> $TMP/$name.log
        echo "== $name" >> stats.txt
        grep -E '^(Got all|Allocated|# multi-mappings that|After allocating)' $TMP/$name.log | sed -E 's/ in [0-9.e+-]+s\././' >> stats.txt; }
SMPE="-1 $TMP/sm_read1.fq -2 $TMP/sm_read2.fq"
run q0 bed sm $SMPE -q 0
run n4q0 bed sm $SMPE -n 4 -q 0
run n4q0_d200 bed sm $SMPE -n 4 -q 0 --multi-mapping-allocation-distance 200
run n4q0_d5000 bed sm $SMPE -n 4 -q 0 --multi-mapping-allocation-distance 5000
run n4q0_s5 bed sm $SMPE -n 4 -q 0 --multi-mapping-allocation-seed 5
run n4q0_s0 bed sm $SMPE -n 4 -q 0 --multi-mapping-allocation-seed 0
run n4q0_sm1 bed sm $SMPE -n 4 -q 0 --multi-mapping-allocation-seed -1
run n4q0_dedup_tn5 bed sm $SMPE -n 4 -q 0 --remove-pcr-duplicates --Tn5-shift
run n8q0 bed sm $SMPE -n 8 -q 0
run n4 bed sm $SMPE -n 4
run n4q0_tagalign tagalign sm $SMPE -n 4 -q 0 --TagAlign
run se_n3q0 bed sm -1 $TMP/sm_read1.fq -n 3 -q 0
run se_n4q0_d200 bed sm -1 $TMP/sm_read1.fq -n 4 -q 0 --multi-mapping-allocation-distance 200
SCWL="-b $TMP/sc_barcode.fq --barcode-whitelist $SC/whitelist.txt"
run sc_n4q0 bed sc -1 $TMP/sc_read1.fq -2 $TMP/sc_read2.fq $SCWL -n 4 -q 0 --remove-pcr-duplicates --Tn5-shift --trim-adapters -l 2000
run sc_se_n4q0 bed sc -1 $TMP/sc_read1.fq $SCWL -n 4 -q 0 --remove-pcr-duplicates
for f in *.bed *.tagalign; do md5sum $f; done | awk '{print $1, $2}' > md5.txt
gzip -9n *.bed *.tagalign
# low-memory mode: accepted and ignored
$REF -x $TMP/sm.index -r $TMP/sm_ref.fa -t 1 --preset chip --allocate-multi-mappings $SMPE -o $TMP/chip.bed 2> /dev/null
gzip -dc $SM/chip.bed.gz | cmp - $TMP/chip.bed
# no multi-mapping: the reference aborts (exit 134)
head -12 $TMP/sm_read1.fq > $TMP/few1.fq; head -12 $TMP/sm_read2.fq > $TMP/few2.fq
set +e
$REF -x $TMP/sm.index -r $TMP/sm_ref.fa -t 1 --allocate-multi-mappings -q 0 -1 $TMP/few1.fq -2 $TMP/few2.fq -o $TMP/few.bed 2> /dev/null
rc=$?
set -e
test $rc -ne 0
echo "synth_allocate: $(ls *.gz | wc -l) outputs; the first three pairs: exit $rc"
