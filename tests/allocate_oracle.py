"""Test infrastructure: the oracle's in-memory post-processing with --allocate-multi-mappings (chromap.h:1322-1355): Tn5, sort,
dedup (oracle/, MAPQ filter at 0), the allocation of tests/allocate_oracle.h (built into a shared object in a temporary
directory), then sort and MAPQ filter again (oracle/, dedup and Tn5 off)."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle_py as orc

HERE = os.path.dirname(os.path.abspath(__file__))

SHIM = r'''
#include "%s"
extern "C" int orc_allocate(const orc_alloc_record *recs, uint64_t n, uint32_t n_seq, int32_t d, int32_t seed, uint8_t *keep, orc_alloc_stats *st) {
  return orc_allocate_flags(recs, n, n_seq, d, seed, keep, st);
}
'''

STATS = ("n_multi", "n_allocated", "n_without_overlap", "n_draws", "n_uni_after", "n_multi_after")


class Stats(C.Structure):
    _fields_ = [(f, C.c_uint64) for f in STATS]


def load(tmp_dir):
    """Builds the allocation restatement in tmp_dir; returns the ctypes library."""
    src = os.path.join(str(tmp_dir), "allocate_oracle.cc")
    so = os.path.join(str(tmp_dir), "liballocate_oracle.so")
    open(src, "w").write(SHIM % os.path.join(HERE, "allocate_oracle.h"))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    L = C.CDLL(so)
    L.orc_allocate.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(Stats)]
    return L


def _postprocess(params, recs, bcs):
    if bcs is not None:
        return orc.postprocess_bc(params, recs, bcs)
    return (orc.postprocess_se(params, recs) if params.single_end else orc.postprocess(params, recs)), None


def allocate(L, params, recs, bcs, n_seq, distance=0, seed=11):
    """(records, barcode keys or None, stats dict, or None when there is no multi-mapping: the reference aborts)."""
    p1 = orc.make_params()
    for f, _ in orc.Params._fields_:
        setattr(p1, f, getattr(params, f))
    p1.mapq_threshold = 0
    r1, b1 = _postprocess(p1, recs, bcs)
    r1 = np.ascontiguousarray(r1)
    keep = np.zeros(len(r1), dtype=np.uint8)
    st = Stats()
    if L.orc_allocate(r1.ctypes.data, len(r1), n_seq, distance, seed, keep.ctypes.data, C.byref(st)) != 0:
        return None
    sel = keep.astype(bool)
    p2 = orc.make_params()
    for f, _ in orc.Params._fields_:
        setattr(p2, f, getattr(params, f))
    p2.remove_pcr_duplicates = 0
    p2.tn5_shift = 0
    r2, b2 = _postprocess(p2, r1[sel], b1[sel] if b1 is not None else None)
    return r2, b2, {f: int(getattr(st, f)) for f in STATS}


def golden_stats(path):
    """stats.txt -> {case: dict of the four log lines' counts}."""
    return golden_stats_text(open(path).read())


def golden_stats_text(text):
    """The same for text ("== case" lines, then the log lines of that case)."""
    import re
    out, name = {}, None
    for line in text.split("\n"):
        line = line.strip()
        if line.startswith("== "):
            name = line[3:]
            out[name] = {}
            continue
        nums = [int(x) for x in re.findall(r"\d+", line)]
        if line.startswith("Got all"):
            out[name]["n_multi"] = nums[0]
        elif line.startswith("Allocated"):
            out[name]["n_allocated"] = nums[0]
        elif line.startswith("# multi-mappings"):
            out[name]["n_without_overlap"] = nums[0]
        elif line.startswith("After allocating"):
            out[name]["n_uni_after"], out[name]["n_multi_after"] = nums[0], nums[1]
    return out


# The cases of tests/golden/make_golden_allocate.sh: data set, single-end, barcoded, oracle parameters, distance, seed, text
# format, and the chromap command line (without the files and --allocate-multi-mappings)
def _case(data, se, bc, kw, d=0, s=11, fmt="bed", args=()):
    return dict(data=data, se=se, bc=bc, kw=kw, distance=d, seed=s, fmt=fmt, args=list(args))


N4 = dict(max_num_best_mappings=4, mapq_threshold=0)
CASES = {
    "q0": _case("synth_small", False, False, dict(mapq_threshold=0), args=["-q", "0"]),
    "n4q0": _case("synth_small", False, False, N4, args=["-n", "4", "-q", "0"]),
    "n4q0_d200": _case("synth_small", False, False, N4, d=200, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-distance", "200"]),
    "n4q0_d5000": _case("synth_small", False, False, N4, d=5000, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-distance", "5000"]),
    "n4q0_s5": _case("synth_small", False, False, N4, s=5, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-seed", "5"]),
    "n4q0_s0": _case("synth_small", False, False, N4, s=0, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-seed", "0"]),
    "n4q0_sm1": _case("synth_small", False, False, N4, s=-1, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-seed", "-1"]),
    "n4q0_dedup_tn5": _case("synth_small", False, False, dict(N4, remove_pcr_duplicates=1, tn5_shift=1),
                            args=["-n", "4", "-q", "0", "--remove-pcr-duplicates", "--Tn5-shift"]),
    "n8q0": _case("synth_small", False, False, dict(max_num_best_mappings=8, mapq_threshold=0), args=["-n", "8", "-q", "0"]),
    "n4": _case("synth_small", False, False, dict(max_num_best_mappings=4), args=["-n", "4"]),
    "n4q0_tagalign": _case("synth_small", False, False, N4, fmt="tagalign", args=["-n", "4", "-q", "0", "--TagAlign"]),
    "se_n3q0": _case("synth_small", True, False, dict(max_num_best_mappings=3, mapq_threshold=0), args=["-n", "3", "-q", "0"]),
    "se_n4q0_d200": _case("synth_small", True, False, N4, d=200, args=["-n", "4", "-q", "0", "--multi-mapping-allocation-distance", "200"]),
    "sc_n4q0": _case("synth_sc", False, True, dict(N4, remove_pcr_duplicates=1, tn5_shift=1, trim_adapters=1, max_insert_size=2000),
                     args=["-n", "4", "-q", "0", "--remove-pcr-duplicates", "--Tn5-shift", "--trim-adapters", "-l", "2000"]),
    "sc_se_n4q0": _case("synth_sc", True, True, dict(N4, remove_pcr_duplicates=1), args=["-n", "4", "-q", "0", "--remove-pcr-duplicates"]),
}


def _barcodes(path):
    import gzip
    lines = gzip.open(path).read().split(b"\n")
    return np.frombuffer(b"".join(lines[1::4]), dtype=np.uint8), np.frombuffer(b"".join(lines[3::4]), dtype=np.uint8), len(lines[1])


def oracle_records(golden_dir, case):
    """The oracle's mapping of a case (one batch, like the reference at -t 1): (reference, params, records, barcode keys or
    None, barcode length)."""
    from tests.util import load_pairs
    c = CASES[case]
    d = os.path.join(golden_dir, c["data"])
    ref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    idx = orc.Index(ref=ref, k=17, w=7)
    s1, o1, s2, o2 = load_pairs(d)
    p = orc.make_params("", single_end=int(c["se"]), **c["kw"])
    if not c["bc"]:
        recs = orc.map_reads_se(p, idx, ref, s1, o1) if c["se"] else orc.map_pairs(p, idx, ref, s1, o1, s2, o2)[0]
        return ref, p, recs, None, 0
    bcs, quals, bc_len = _barcodes(os.path.join(d, "barcode.fq.gz"))
    wl = orc.Whitelist(os.path.join(d, "whitelist.txt"), bc_len)
    wl.sample(bcs)
    if c["se"]:
        recs, keys, _ = orc.map_reads_se_bc(p, idx, ref, s1, o1, bcs, quals, bc_len, whitelist=wl)
    else:
        recs, keys, _ = orc.map_pairs_bc(p, idx, ref, s1, o1, s2, o2, bcs, quals, bc_len, whitelist=wl)
    return ref, p, recs, keys, bc_len


def format_text(ref, case, recs, keys, bc_len):
    fmt = CASES[case]["fmt"]
    if keys is not None:
        return orc.format_bed_bc(ref, recs, keys, bc_len)
    return orc.format_tagalign(ref, recs) if fmt == "tagalign" else orc.format_bed(ref, recs)
