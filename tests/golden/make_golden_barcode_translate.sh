#!/bin/bash
# Regenerates tests/golden/synth_barcode_translate/ from the UNMODIFIED reference binary (oracle/_ref/chromap, built by
# oracle/Makefile): --barcode-translate cases.  The tables are derived from synth_sc/whitelist.txt without randomness and
# committed gzipped; the synth_sc (and, for the bulk case, synth_small) inputs are used as they are.  Identity cases are
# compared with cmp against other outputs; the reference's exit status and message for a missing barcode are asserted.
set -e
cd "$(dirname "$0")"
GOLDEN=$(pwd)
REF=$(cd ../.. && pwd)/oracle/_ref/chromap
SC=$GOLDEN/synth_sc
SMALL=$GOLDEN/synth_small
RF=$GOLDEN/synth_read_format
rm -rf synth_barcode_translate && mkdir -p synth_barcode_translate
cd synth_barcode_translate
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
mkdir -p $TMP/sc $TMP/small
for f in ref.fa read1.fq read2.fq barcode.fq; do gzip -dc $SC/$f.gz > $TMP/sc/$f; done
for f in ref.fa read1.fq read2.fq; do gzip -dc $SMALL/$f.gz > $TMP/small/$f; done
gzip -dc $RF/bc24.fq.gz > $TMP/sc/bc24.fq
python3 - "$SC/whitelist.txt" <<'EOF'
import itertools, sys
wl = open(sys.argv[1]).read().split()
rc = lambda s: s.translate(str.maketrans("ACGT", "TGCA"))[::-1]
def write(path, lines, final_newline=True):
    open(path, "w").write("\n".join(lines) + ("\n" if final_newline else ""))
# 16 -> 16, comma-separated, like the 10x Multiome ATAC -> gene-expression table
write("rc16.txt", ["%s,%s" % (rc(w), w) for w in wl])
# tab-separated, names of varying length; every 7th FROM in lower case; the FROM of entry 5 again at the end with another
# name (the later line wins); entries no barcode maps to; no newline after the last line
names = ["cell_%d%s\t%s" % (i, "x" * (i % 5), w.lower() if i % 7 == 0 else w) for i, w in enumerate(wl)]
names += ["unused_%d\t%s" % (i, "".join(p)) for i, p in enumerate(itertools.islice(itertools.product("ACGT", repeat=16), 0, 4000, 400))]
names.append("second_name_of_5\t" + wl[5])
write("names.txt", names, final_newline=False)
# every 8-base half of a whitelist entry (16 = 2 x 8: fields X-Y)
halves = sorted({w[a:a + 8] for w in wl for a in (0, 8)})
write("half8.txt", ["h%d,%s" % (i, h) for i, h in enumerate(halves)])
# all 5-mers (16 = 3 x 5 + 1: the first base is dropped, three fields)
write("all5.txt", ["%s%d,%s" % ("".join(p).lower(), i, "".join(p)) for i, p in enumerate(itertools.product("ACGT", repeat=5))])
# L = 20 > 16: no segment, every field is empty
write("long20.txt", ["L%d,%sACGT" % (i, w) for i, w in enumerate(wl)])
EOF
gzip -9 -n rc16.txt half8.txt all5.txt long20.txt
gzip -9 -n names.txt
$REF -i -r $TMP/sc/ref.fa -o $TMP/sc/ref.index 2> /dev/null
$REF -i -r $TMP/small/ref.fa -o $TMP/small/ref.index 2> /dev/null
WL="--barcode-whitelist $SC/whitelist.txt"
sc() { name=$1; shift; $REF -x $TMP/sc/ref.index -r $TMP/sc/ref.fa -t 1 "$@" -o $name 2> /dev/null; }
PE="-1 $TMP/sc/read1.fq -2 $TMP/sc/read2.fq -b $TMP/sc/barcode.fq"
SE="-1 $TMP/sc/read1.fq -b $TMP/sc/barcode.fq"
sc pe_rc16.bed --preset atac $WL $PE --barcode-translate rc16.txt.gz
sc se_rc16.bed --preset atac $WL $SE --barcode-translate rc16.txt.gz
sc se_inmem_rc16.bed -q 0 --remove-pcr-duplicates --Tn5-shift $WL $SE --barcode-translate rc16.txt.gz
sc pe_names.bed --preset atac $WL $PE --barcode-translate names.txt.gz
sc pe_half8.bed --preset atac $WL $PE --barcode-translate half8.txt.gz
sc pe_all5_nowl.bed --preset atac $PE --barcode-translate all5.txt.gz
sc pe_all5_notinwl.bed --preset atac $WL --output-mappings-not-in-whitelist $PE --barcode-translate all5.txt.gz
sc pe_long20.bed --preset atac $WL $PE --barcode-translate long20.txt.gz
# identity cases: the barcode inside a longer read gives the same fields; a bulk run loads the table and ignores it
sc $TMP/o.bed --preset atac $WL -1 $TMP/sc/read1.fq -2 $TMP/sc/read2.fq -b $TMP/sc/bc24.fq --read-format bc:8:23 --barcode-translate rc16.txt.gz
cmp pe_rc16.bed $TMP/o.bed
$REF --preset chip -x $TMP/small/ref.index -r $TMP/small/ref.fa -1 $TMP/small/read1.fq -2 $TMP/small/read2.fq -t 1 --barcode-translate rc16.txt.gz -o $TMP/o.bed 2> /dev/null
gzip -dc $SMALL/chip.bed.gz | cmp - $TMP/o.bed
# the table without the commonest output barcode: the reference stops with status 255 and its message
top=$(cut -f4 pe_rc16.bed | sort | uniq -c | sort -k1,1nr -k2,2 | head -1 | awk '{print $2}')
gzip -dc rc16.txt.gz | grep -v "^$top," | gzip -9 -n > missing_rc16.txt.gz
test $(gzip -dc missing_rc16.txt.gz | wc -l) -eq $(( $(gzip -dc rc16.txt.gz | wc -l) - 1 ))
set +e
$REF --preset atac $WL $PE --barcode-translate missing_rc16.txt.gz -x $TMP/sc/ref.index -r $TMP/sc/ref.fa -t 1 -o $TMP/o.bed 2> $TMP/err.txt
status=$?
set -e
test $status -eq 255
grep -qx "Barcode does not exist in the translation table." $TMP/err.txt
md5sum *.bed > md5.txt
gzip -9 -n *.bed
