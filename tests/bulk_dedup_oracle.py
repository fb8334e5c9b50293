"""Test infrastructure: the reference's bulk-level duplicate removal of barcoded BED (tests/golden/make_golden_bulk_dedup.sh)
restated on top of oracle/oracle_py.py.  The records and barcode keys come from the oracle's barcoded mapping (map_pairs_bc /
map_reads_se_bc) with the whitelist sampled as the reference does; `merge` transcribes the merge loop of
ProcessAndOutputMappingsInLowMemory (mapping_writer.h:166-376) with FindBestMappingIndexFromDuplicates (:126-163), one record at
a time; the BED text (mapping_writer.cc:127-137) is written here in Python."""
import functools
import gzip
import os

import numpy as np

from oracle import oracle_py as orc
from tests import bc_error2_oracle as bce
from tests import translate_oracle as tro
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SC = os.path.join(GOLDEN, "synth_sc")
OUT = os.path.join(GOLDEN, "synth_bulk_dedup")
WL = os.path.join(SC, "whitelist.txt")
RC16 = os.path.join(GOLDEN, "synth_barcode_translate", "rc16.txt.gz")

# output: (preset, parameter overrides, single-end, --barcode-translate table); every run gives --barcode-whitelist
RUNS = {
    "pe_chip": ("chip", {}, False, None),
    "se_chip": ("chip", {}, True, None),
    "pe_q0": ("", dict(low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=0), False, None),
    "se_q0": ("", dict(low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=0), True, None),
    "pe_atac_bulk": ("atac", {}, False, None),
    "pe_chip_rc16": ("chip", {}, False, RC16),
    "pe_inmem_q0": ("", dict(remove_pcr_duplicates=1, mapq_threshold=0), False, None),
}


def params(name):
    preset, kw, se, _ = RUNS[name]
    return orc.make_params(preset, single_end=int(se), **kw)


def bulk_level(name):
    """The runs that remove duplicates at bulk level: low-memory ones (in memory the level plays no part)."""
    p = params(name)
    return bool(p.low_memory_mode and p.remove_pcr_duplicates)


@functools.lru_cache(maxsize=1)
def setup():
    ref = orc.Reference(os.path.join(SC, "ref.fa.gz"))
    bcs, quals, bc_len = bce.read_barcodes(os.path.join(OUT, "barcode.fq.gz"))
    wl = orc.Whitelist(WL, bc_len)
    wl.sample(bcs)
    return ref, orc.Index(ref=ref, k=17, w=7), load_pairs(OUT), wl, (bcs, quals, bc_len)


def whitelist():
    """(keys, counts) of the whitelist with the sampled abundances."""
    keys, counts, _ = setup()[3].arrays()
    return keys, counts


@functools.lru_cache(maxsize=None)
def records(name):
    """The oracle's barcoded records and keys of the run, before post-processing."""
    ref, index, (s1, o1, s2, o2), wl, (bcs, quals, bc_len) = setup()
    p = params(name)
    if RUNS[name][2]:
        recs, keys, _ = orc.map_reads_se_bc(p, index, ref, s1, o1, bcs, quals, bc_len, wl)
    else:
        recs, keys, _ = orc.map_pairs_bc(p, index, ref, s1, o1, s2, o2, bcs, quals, bc_len, wl)
    return recs, keys


def _tn5(r, se):
    if se:  # bed_mapping.h:97-103
        if r["direction"] == 1:
            r["fragment_start"] += 4
        else:
            r["fragment_length"] = (int(r["fragment_length"]) - 5) & 0xFFFF
    else:  # bed_mapping.h:225-230
        r["fragment_start"] += 4
        r["positive_alignment_length"] = (int(r["positive_alignment_length"]) - 4) & 0xFFFF
        r["fragment_length"] = (int(r["fragment_length"]) - 9) & 0xFFFF
        r["negative_alignment_length"] = (int(r["negative_alignment_length"]) - 5) & 0xFFFF


def merge(p, abundance, recs, keys):
    """ProcessAndOutputMappingsInLowMemory at bulk level over barcoded records: (records, keys) written, in order.
    `abundance` maps a barcode key to its whitelist count (KeyError for a barcode outside it, where the reference reads out of
    bounds)."""
    se = bool(p.single_end)
    order = sorted(range(len(recs)), key=lambda i: (int(recs[i]["rid"]), int(recs[i]["fragment_start"]), int(recs[i]["fragment_length"]), int(keys[i]),
                                                  int(recs[i]["mapq"]), int(recs[i]["direction"]), int(recs[i]["is_unique"]), int(recs[i]["read_id"])))
    pos = lambda i: (int(recs[i]["fragment_start"]),) if se else (int(recs[i]["fragment_start"]), int(recs[i]["fragment_length"]))  # IsSamePosition
    eq = lambda a, b: keys[a] == keys[b] and pos(a) == pos(b)  # operator==
    out_r, out_k = [], []
    dups = []  # temp_dups_for_bulk_level_dedup: [record index, num_dups_]

    def find_best():
        best = 0
        best_ab = abundance[int(keys[dups[0][0]])]
        for k in range(1, len(dups)):
            ab = abundance[int(keys[dups[k][0]])]
            if dups[k][1] > dups[best][1] or (dups[k][1] == dups[best][1] and ab > best_ab):
                best, best_ab = k, ab
        return dups[best][0]

    def append(i, n_dups):
        r = recs[i].copy()
        r["num_dups"] = min(255, n_dups)
        if p.tn5_shift:
            _tn5(r, se)
        out_r.append(r)
        out_k.append(keys[i])

    last_rid, last, n_last = None, None, 0
    for t, cur in enumerate(order):
        rid = int(recs[cur]["rid"])
        duplicated = t > 0 and rid == last_rid and (eq(cur, last) or pos(cur) == pos(last))
        if p.remove_pcr_duplicates and duplicated:
            n_last += 1
            if dups and eq(cur, dups[-1][0]):
                dups[-1] = [cur, 1 + 1]  # the stored record becomes cur (num_dups_ 1), then += 1
            else:
                dups.append([cur, 1])
            if recs[cur]["mapq"] > recs[last]["mapq"]:
                last = cur
        else:
            if t > 0:
                last = find_best()
                dups = []
                if recs[last]["mapq"] >= p.mapq_threshold:
                    append(last, n_last)
            last, last_rid, n_last = cur, rid, 1
            dups.append([cur, 1])
    if order and recs[last]["mapq"] >= p.mapq_threshold:  # the last group: its threshold is tested before the best entry is found
        append(find_best(), n_last)
    return (np.array(out_r, dtype=recs.dtype) if out_r else recs[:0].copy()), np.array(out_k, dtype=np.uint64)


def bed_text(ref_names, recs, keys, bc_len, translation=None):
    lines = []
    for r, k in zip(recs, keys):
        field = tro.translate(translation, int(k), bc_len) if translation is not None else \
            "".join("ACGT"[(int(k) >> (2 * (bc_len - 1 - j))) & 3] for j in range(bc_len))
        if isinstance(field, bytes):
            field = field.decode()
        s = int(r["fragment_start"])
        lines.append("%s\t%d\t%d\t%s\t%d\n" % (ref_names[int(r["rid"])], s, (s + int(r["fragment_length"])) & 0xFFFFFFFF, field, int(r["num_dups"])))
    return "".join(lines).encode()


def ref_names():
    from tests.util import read_fasta
    return read_fasta(os.path.join(SC, "ref.fa.gz"))[0]


def run(name):
    """The oracle's BED text of the run."""
    recs, keys = records(name)
    p = params(name)
    bc_len = setup()[4][2]
    if bulk_level(name):
        wk, wc = whitelist()
        out_r, out_k = merge(p, dict(zip(wk.tolist(), wc.tolist())), recs, keys)
    else:
        out_r, out_k = orc.postprocess_bc(p, recs, keys)
    tr = RUNS[name][3]
    return bed_text(ref_names(), out_r, out_k, bc_len, tro.load_translation(gzip.open(tr).read()) if tr else None)


def golden(name):
    return gzip.open(os.path.join(OUT, name + ".bed.gz")).read()
