"""Test infrastructure: the reference's --SAM with cell barcodes (tests/golden/make_golden_sam_bc.sh) restated on top of
oracle/oracle_py.py.  The cores come from the oracle's SAM mapping (orc_map_sam_cores) behind the barcode gate of
orc_map_pairs_bc / orc_map_reads_se_bc (chromap.h:897-909, 392-409): a read whose barcode is neither in the whitelist nor
corrected is given to the mapper as an empty read, which maps to nothing and draws nothing from the batch chunk's generator,
as the reference's `continue` does.  The text is SAMMapping's order, duplicate test and MAPQ filter with the cell barcode
(sam_mapping.h:188-199, mapping_processor.h:161-202, mapping_writer.h:166-376) and the lines of mapping_writer.cc:312-356,
written here in Python, independently of the library's writers."""
import functools
import gzip
import os

import numpy as np

from oracle import oracle_py as orc
from tests import bc_error2_oracle as bce
from tests import translate_oracle as tro
from tests.util import read_fastq_records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SC = os.path.join(GOLDEN, "synth_sc")
BE = os.path.join(GOLDEN, "synth_bc_error2")
TR = os.path.join(GOLDEN, "synth_barcode_translate")
OUT = os.path.join(GOLDEN, "synth_sam_bc")
WL = os.path.join(SC, "whitelist.txt")
BATCH = 500000

# output: (preset, parameter overrides, single-end, barcode file, whitelist, --bc-error-threshold,
#          --output-mappings-not-in-whitelist, --barcode-translate table)
RUNS = {
    "pe_atac": ("atac", {}, False, "barcode.fq.gz", WL, 1, False, None),
    "se_atac": ("atac", {}, True, "barcode.fq.gz", WL, 1, False, None),
    "pe_q0dedup": ("", dict(mapq_threshold=0, remove_pcr_duplicates=1), False, "barcode.fq.gz", WL, 1, False, None),
    "se_q0dedup": ("", dict(mapq_threshold=0, remove_pcr_duplicates=1), True, "barcode.fq.gz", WL, 1, False, None),
    "pe_nowl": ("atac", {}, False, "barcode.fq.gz", None, 1, False, None),
    "pe_notinwl": ("atac", {}, False, "barcode.fq.gz", WL, 1, True, None),
    "pe_n3q0": ("", dict(max_num_best_mappings=3, mapq_threshold=0), False, "barcode.fq.gz", WL, 1, False, None),
    "pe_bcerr2": ("atac", {}, False, os.path.join(BE, "barcode.fq.gz"), os.path.join(BE, "dense.txt.gz"), 2, False, None),
    "pe_rc16": ("atac", {}, False, "barcode.fq.gz", WL, 1, False, os.path.join(TR, "rc16.txt.gz")),
    "pe_half8": ("atac", {}, False, "barcode.fq.gz", WL, 1, False, os.path.join(TR, "half8.txt.gz")),
}


@functools.lru_cache(maxsize=1)
def setup():
    """The synth_sc reference, its index and reads [(name, bases, qualities)] of both files."""
    ref = orc.Reference(os.path.join(SC, "ref.fa.gz"))
    return ref, orc.Index(ref=ref, k=17, w=7), read_fastq_records(os.path.join(SC, "read1.fq.gz")), read_fastq_records(os.path.join(SC, "read2.fq.gz"))


def params(name):
    preset, kw, se, _, _, _, _, _ = RUNS[name]
    return orc.make_params(preset, single_end=int(se), **kw)


def barcode_gate(name):
    """(barcode key, passes the gate) of every read of the run, and the barcode length."""
    _, _, _, bc_path, wl_path, err, notinwl, _ = RUNS[name]
    bcs, quals, bc_len = bce.read_barcodes(bc_path if os.path.isabs(bc_path) else os.path.join(SC, bc_path))
    if wl_path is None:
        keys = np.array([tro._seed(bytes(bcs[i * bc_len:(i + 1) * bc_len])) for i in range(len(bcs) // bc_len)], dtype=np.uint64)
        return keys, np.ones(len(keys), dtype=bool), bc_len
    wl = orc.Whitelist(wl_path, bc_len)
    wl.sample(bcs)
    keys, ok, _, _ = bce.correct_barcodes(wl, err, 0.9, bcs, quals, bc_len, notinwl)
    return keys, ok.astype(bool), bc_len


def cores_and_keys(p, index, ref, reads1, reads2, keys, ok):
    """SAM cores of the reads that pass the gate, one reference batch at a time, and each core's barcode key."""
    cores = []
    for b0 in range(0, len(reads1), BATCH):
        sel = range(b0, min(len(reads1), b0 + BATCH))
        s1 = [reads1[i][1] if ok[i] else b"" for i in sel]
        off1 = np.zeros(len(s1) + 1, dtype=np.uint32); off1[1:] = np.cumsum([len(x) for x in s1])
        seq1 = np.frombuffer(b"".join(s1), dtype=np.uint8)
        seq2 = off2 = None
        if reads2 is not None:
            s2 = [reads2[i][1] if ok[i] else b"" for i in sel]
            off2 = np.zeros(len(s2) + 1, dtype=np.uint32); off2[1:] = np.cumsum([len(x) for x in s2])
            seq2 = np.frombuffer(b"".join(s2), dtype=np.uint8)
        cores.append(orc.map_sam_cores(p, index, ref, seq1, off1, seq2, off2, first_read_id=b0))
    cores = np.concatenate(cores)
    return cores, keys[cores["read_id"]]


def _md(ref_seq, pos, cigar, seq):
    nm, nmatch, md, r, g = 0, 0, b"", 0, pos
    for c in cigar:
        op, ol = c & 0xF, c >> 4
        if op == 0:
            for _ in range(ol):
                gb, sb = int(ref_seq[g]), seq[r]
                if gb == sb or gb - ord("a") + ord("A") == sb:
                    nmatch += 1
                else:
                    nm += 1; md += b"%d" % nmatch + bytes([gb]); nmatch = 0
                r += 1; g += 1
        elif op == 1:
            nm += ol; r += ol
        else:
            nm += ol; md += b"%d^" % nmatch + bytes(ref_seq[g:g + ol]); nmatch = 0; g += ol
    return nm, md + b"%d" % nmatch


_COMP = {ord("A"): b"T", ord("a"): b"T", ord("C"): b"G", ord("c"): b"G", ord("G"): b"C", ord("g"): b"C", ord("T"): b"A", ord("t"): b"A"}


def format_sam(p, ref, cores, keys, reads1, reads2, bc_len, translation=None):
    """@SQ header + lines; keys None: bulk.  Raises translate_oracle.BarcodeMissing where the reference exits."""
    pe = reads2 is not None
    lines = []
    for ci, c in enumerate(cores):
        bc = int(keys[ci]) if keys is not None else 0
        if not pe:
            lines.append((int(c["rid"]), int(c["pos"][0]), bc, -1, 0, 0, int(c["mapq"]), int(c["read_id"]),
                          ci, 0, (0 if c["strand"][0] else 16) | (256 if c["secondary"] else 0), 0))
            continue
        f1, f2 = 3 | 64, 3 | 128
        if not c["strand"][0]: f1 |= 16; f2 |= 32
        if not c["strand"][1]: f1 |= 32; f2 |= 16
        if c["secondary"]: f1 |= 256; f2 |= 256
        tlen = int(c["end"][1]) - int(c["pos"][0]) + 1 if c["strand"][0] else int(c["end"][0]) - int(c["pos"][1]) + 1
        for mate, f in ((0, f1), (1, f2)):
            t = tlen if c["strand"][mate] else -tlen
            lines.append((int(c["rid"]), int(c["pos"][mate]), bc, int(c["rid"]), int(c["pos"][1 - mate]), f & 64, int(c["mapq"]), int(c["read_id"]), ci, mate, f, t))
    lines.sort(key=lambda l: l[:8])  # stable: ties keep the expansion order
    keep = []
    i = 0
    while i < len(lines):
        j, k = i + 1, i
        if p.remove_pcr_duplicates:
            while j < len(lines) and lines[j][:6] == lines[j - 1][:6]:  # (rid, pos, barcode, mrid, mpos, read 1)
                if not p.low_memory_mode or lines[j][6] > lines[k][6]:
                    k = j
                j += 1
        if lines[k][6] >= p.mapq_threshold:
            keep.append(lines[k])
        i = j
    out = [b"@SQ\tSN:%s\tLN:%d\n" % (ref.names[r].encode(), ref.lengths[r]) for r in range(ref.n)]
    seqs = {}
    for rid, pos, bc, mrid, mpos, _, mapq, read_id, ci, mate, flag, tlen in keep:
        c = cores[ci]
        name, rseq, rqual = (reads2 if mate else reads1)[read_id]
        cig = [int(x) for x in c["cigar"][mate][:c["n_cigar"][mate]]]
        rl = sum(x >> 4 for x in cig if x & 0xF != 2)
        plus = bool(c["strand"][mate])
        seq = rseq[:rl] if plus else b"".join(_COMP.get(x, b"N") for x in reversed(rseq[:rl]))
        qual = (rqual if plus else rqual[::-1])[:rl]
        if rid not in seqs:
            seqs[rid] = ref.seq(rid)
        nm, md = _md(seqs[rid], pos, cig, seq)
        cigar = b"".join(b"%d%s" % (x >> 4, b"MIDNSHP=XB"[x & 0xF:(x & 0xF) + 1]) for x in cig) or b"*"
        mate_field = b"*" if mrid < 0 else b"="
        line = b"\t".join([name, b"%d" % flag, ref.names[rid].encode(), b"%d" % (pos + 1), b"%d" % mapq, cigar, mate_field,
                           b"%d" % (0 if mrid < 0 else mpos + 1), b"%d" % tlen, seq, qual, b"NM:i:%d" % nm, b"MD:Z:" + md])
        if keys is not None:
            field = tro.translate(translation, bc, bc_len) if translation else bytes(b"ACGT"[(bc >> (2 * (bc_len - 1 - j))) & 3] for j in range(bc_len))
            line += b"\tCB:Z:" + field
        out.append(line + b"\n")
    return b"".join(out)


def run(name):
    """The run's whole SAM file, as the reference writes it."""
    ref, index, reads1, reads2 = setup()
    _, _, se, _, _, _, _, tr_path = RUNS[name]
    p = params(name)
    keys, ok, bc_len = barcode_gate(name)
    cores, ck = cores_and_keys(p, index, ref, reads1, None if se else reads2, keys, ok)
    translation = tro.load_translation(gzip.open(tr_path).read()) if tr_path else None
    return format_sam(p, ref, cores, ck, reads1, None if se else reads2, bc_len, translation)
