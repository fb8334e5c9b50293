"""Test infrastructure: the oracle's scATAC mapping at --bc-error-threshold 2 on the synth_bc_error2 fixtures
(tests/golden/make_golden_bc_error2.sh).  oracle_py.map_pairs_bc / map_reads_se_bc fix the barcode options at the
reference's defaults (threshold 1, probability 0.9, mappings outside the whitelist dropped); this module sets them through
orc_mapper_set_barcodes on top of oracle/oracle_py.py."""
import ctypes as C
import functools
import gzip
import os

import numpy as np

from oracle import oracle_py as orc
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SC = os.path.join(ROOT, "tests", "golden", "synth_sc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "synth_bc_error2")

# output: (barcode file, whitelist file, single-end, --bc-probability-threshold, --output-mappings-not-in-whitelist); all
# --preset atac --bc-error-threshold 2
RUNS = {
    "pe_wl": (os.path.join(GOLDEN, "barcode.fq.gz"), os.path.join(SC, "whitelist.txt"), False, 0.9, False),
    "pe_dense": (os.path.join(GOLDEN, "barcode.fq.gz"), os.path.join(GOLDEN, "dense.txt.gz"), False, 0.9, False),
    "pe_dense_p04": (os.path.join(GOLDEN, "barcode.fq.gz"), os.path.join(GOLDEN, "dense.txt.gz"), False, 0.4, False),
    "pe_dense_notinwl": (os.path.join(GOLDEN, "barcode.fq.gz"), os.path.join(GOLDEN, "dense.txt.gz"), False, 0.9, True),
    "se_dense": (os.path.join(GOLDEN, "barcode.fq.gz"), os.path.join(GOLDEN, "dense.txt.gz"), True, 0.9, False),
    "pe_orig": (os.path.join(SC, "barcode.fq.gz"), os.path.join(SC, "whitelist.txt"), False, 0.9, False),
}


def read_barcodes(path):
    """(bases, qualities, bc_len) of a 4-line FASTQ of equal-length barcodes, as uint8 concatenations."""
    lines = gzip.open(path).read().split(b"\n")
    return np.frombuffer(b"".join(lines[1::4]), dtype=np.uint8), np.frombuffer(b"".join(lines[3::4]), dtype=np.uint8), len(lines[1])


@functools.lru_cache(maxsize=1)
def setup():
    ref = orc.Reference(os.path.join(SC, "ref.fa.gz"))
    return ref, orc.Index(ref=ref, k=17, w=7), load_pairs(SC)


def whitelist(name):
    """The run's whitelist with the abundances of the reference's pre-pass over its barcodes."""
    bc_path, wl_path, _, _, _ = RUNS[name]
    bcs, _, bc_len = read_barcodes(bc_path)
    wl = orc.Whitelist(wl_path, bc_len)
    wl.sample(bcs)
    return wl


def map_bc(params, index, ref, seq1, off1, seq2, off2, barcodes, quals, bc_len, wl, err_threshold=2, prob_threshold=0.9, output_not_in_whitelist=False,
           n_threads=2):
    """orc_map_pairs_bc (seq2 given) or orc_map_reads_se_bc with the barcode options set: (records, barcode keys, [in whitelist, corrected])."""
    L = orc.lib()
    m = L.orc_mapper_create(C.byref(params), index.h, ref.h)
    L.orc_mapper_set_barcodes(m, wl.h, err_threshold, prob_threshold, int(output_not_in_whitelist))
    n = len(off1) - 1
    out = np.zeros(n * params.max_num_best_mappings, dtype=orc.PE_RECORD)
    obc = np.zeros(len(out), dtype=np.uint64)
    st = np.zeros(2, dtype=np.uint64)
    seq1 = np.ascontiguousarray(seq1, dtype=np.uint8); off1 = np.ascontiguousarray(off1, dtype=np.uint32)
    barcodes = np.ascontiguousarray(barcodes, dtype=np.uint8); quals = np.ascontiguousarray(quals, dtype=np.uint8)
    if seq2 is None:
        got = L.orc_map_reads_se_bc(m, n, seq1.ctypes.data, off1.ctypes.data, barcodes.ctypes.data, quals.ctypes.data, bc_len, 0,
                                    out.ctypes.data, obc.ctypes.data, len(out), n_threads, st.ctypes.data)
    else:
        seq2 = np.ascontiguousarray(seq2, dtype=np.uint8); off2 = np.ascontiguousarray(off2, dtype=np.uint32)
        got = L.orc_map_pairs_bc(m, n, seq1.ctypes.data, off1.ctypes.data, seq2.ctypes.data, off2.ctypes.data, barcodes.ctypes.data, quals.ctypes.data,
                                 bc_len, 0, out.ctypes.data, obc.ctypes.data, len(out), n_threads, st.ctypes.data)
    L.orc_mapper_free(m)
    return out[:got], obc[:got], st


def correct_barcodes(wl, err_threshold, prob_threshold, barcodes, quals, bc_len, output_not_in_whitelist=False):
    """CorrectBarcodeAt per barcode (orc_correct_barcode_test): (keys, ok flags, n_in_whitelist, n_corrected)."""
    L = orc.lib()
    f = L.orc_correct_barcode_test
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    b, q = bytes(np.ascontiguousarray(barcodes, dtype=np.uint8)), bytes(np.ascontiguousarray(quals, dtype=np.uint8))
    n = len(b) // bc_len
    keys, ok = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint8)
    k, n_in, n_cor = C.c_uint64(), C.c_uint64(), C.c_uint64()
    for i in range(n):
        r = f(wl.h, err_threshold, prob_threshold, b[i * bc_len:(i + 1) * bc_len], q[i * bc_len:(i + 1) * bc_len], bc_len, C.byref(k), C.byref(n_in), C.byref(n_cor))
        keys[i], ok[i] = k.value, 1 if (r or output_not_in_whitelist) else 0
    return keys, ok, n_in.value, n_cor.value


def random_set(rng, bc_len, n, n_wl, n_full, path):
    """A whitelist file at `path` (random barcodes; entries one and two substitutions from some of them; every neighbour
    within two substitutions of n_full barcodes that are not listed themselves) and n observed barcodes with qualities:
    listed ones with 0 to 2 substitutions and 0 to 3 Ns, the full-neighbourhood barcodes, random ones.  Returns
    (barcodes, quals, sample) as uint8 arrays; `sample` gives the abundances."""
    A = np.frombuffer(b"ACGT", dtype=np.uint8)
    wl = A[rng.integers(0, 4, (n_wl, bc_len))]
    def subs(x, k):
        x = x.copy()
        for row in x:
            for p in rng.choice(bc_len, k, replace=False):
                row[p] = A[(np.searchsorted(A, row[p]) + rng.integers(1, 4)) % 4]
        return x
    wl = np.concatenate([wl, subs(wl[:n_wl // 3], 2), subs(wl[:n_wl // 6], 1)])
    full = A[rng.integers(0, 4, (n_full, bc_len))]
    nb = []
    for b in full:
        for i in range(bc_len):
            for x in A:
                if x == b[i]:
                    continue
                c = b.copy(); c[i] = x; nb.append(c)
                for j in range(i + 1, bc_len):
                    for y in A:
                        if y != b[j]:
                            d = c.copy(); d[j] = y; nb.append(d)
    allwl = np.concatenate([wl] + ([np.array(nb)] if nb else []))
    fs = {bytes(b) for b in full}
    with open(path, "wb") as f:
        f.write(b"".join(bytes(r) + b"\n" for r in allwl if bytes(r) not in fs))
    obs = allwl[rng.integers(0, len(allwl), n)].copy()
    kind = rng.integers(0, 16, n)
    for t, (s, nn) in enumerate([(2, 0), (2, 0), (2, 0), (1, 0), (1, 0), (1, 1), (0, 1), (0, 2), (1, 2), (0, 3)]):
        for i in np.flatnonzero(kind == t):
            row = obs[i]
            pos = rng.choice(bc_len, min(bc_len, s + nn), replace=False)
            for p in pos[:s]:
                row[p] = A[(np.searchsorted(A, row[p]) + rng.integers(1, 4)) % 4]
            row[pos[s:]] = ord("N")
    rnd = kind == 10
    obs[rnd] = A[rng.integers(0, 4, (int(rnd.sum()), bc_len))]
    if n_full:
        fi = np.flatnonzero(kind == 11)
        obs[fi] = full[rng.integers(0, n_full, len(fi))]
    quals = rng.integers(33, 33 + 45, (n, bc_len)).astype(np.uint8)
    sample = allwl[np.where(rng.integers(0, 3, 4 * len(wl)) == 0, rng.integers(0, len(allwl), 4 * len(wl)), rng.integers(0, len(allwl) // 8 + 1, 4 * len(wl)))]
    return obs.ravel(), quals.ravel(), sample.ravel()


def run_oracle(name):
    """The run's BED text (postprocessed, --preset atac) and counters [in whitelist, corrected], from the oracle."""
    bc_path, _, se, prob, out_nw = RUNS[name]
    ref, idx, (s1, o1, s2, o2) = setup()
    bcs, quals, bc_len = read_barcodes(bc_path)
    p = orc.make_params("atac", single_end=int(se))
    recs, obc, st = map_bc(p, idx, ref, s1, o1, None if se else s2, None if se else o2, bcs, quals, bc_len, whitelist(name), 2, prob, out_nw)
    r2, b2 = orc.postprocess_bc(p, recs, obc)
    return orc.format_bed_bc(ref, r2, b2, bc_len), st
