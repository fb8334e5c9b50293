"""Runs that cross reference-batch, taskloop-chunk and lane boundaries inside one `cmx_map_batch_pe` call, against the oracle.

A call is cut into reference batches of `batch_size` pairs, the batches into up to four lanes (contiguous groups of whole
batches, each on its own host thread and streams), host input goes up in pieces (a quarter batch when `batch_size % 4 == 0`
and `batch_size / 4 >= 32768`, else one batch: batches of 131,072 go up in quarters), barcodes are handed to each lane at its own offset, each lane compacts its
own records, SAM cores and barcode keys, and the lanes' records are put behind one another.  The multi-mapper sampling
restarts at every taskloop chunk of every batch, so batch and chunk boundaries change the output.

The expected records are the oracle's, one oracle call per reference batch with `first_read_id = BASE + b0`, concatenated.
Every configuration is mapped at 1, 3 and 4 lanes, from host buffers into host records and from device buffers into device
records: the records, barcode keys and counters must be the oracle's in every one of those runs.  Floors keep a case from
passing vacuously: at least 3 batches; the overflow tiers 1 and 2 in use (reads longer than `max_read_length`; Hi-C: tier 1,
its 2x150 reads are mapped with `max_read_length` 75); in the batch-size-12,001 runs of paired-end data (records and Hi-C
pairs; the oracle has no single-end trace) a sampled pair (more equally good pairs than `-n`, from the oracle's trace) at
the first pair of every chunk (planted) and within 200 pairs on both sides of every chunk boundary; in barcoded runs a
barcode the oracle corrected in every lane's pairs.

Inputs are made from seeds at test time: a 4.5 Mbp reference with planted exact segment copies (many equally good pairs,
so the sampling decides) and a 300 bp family, reads of 50 to 150 bases (2x150 with chimeric mates for Hi-C), and barcodes
with one and two substitutions and Ns against a whitelist (tests/boundary_inputs.py).

The 15 cases take about 30 s on one H100 80GB HBM3 machine with 8 host CPUs, oracle included."""
import ctypes as C
import functools
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import chromap_b200 as cb
from chromap_b200.binding import Batch, Records
from oracle import oracle_py as orc
from tests.boundary_inputs import ACGT, N_SEQ, make_barcodes, make_reads, reference

pytestmark = pytest.mark.gpu

BASE = 1000003  # first read id of every call
CPUS = os.cpu_count() or 1


@functools.lru_cache(maxsize=1)
def oracle_index():
    seqs, _ = reference()
    oref = orc.Reference(seqs=seqs)
    return oref, orc.Index(ref=oref, k=17, w=7)


# name: (preset, knobs, kind, barcode options (error threshold, output not in whitelist) or None, batch sizes)
# kind: "pe" paired-end records, "se" single-end, "hic" pairs records, "sam_pe" / "sam_se" SAM cores
CONFIGS = {
    "pe_n1": ("", dict(mapq_threshold=0), "pe", None, (12001, 4999, 131072)),   # 131,072: upload pieces of a quarter batch
    "pe_n3": ("", dict(max_num_best_mappings=3, mapq_threshold=0), "pe", None, (12001,)),
    "pe_n8": ("", dict(max_num_best_mappings=8, mapq_threshold=0), "pe", None, (4999,)),
    "atac": ("atac", {}, "pe", None, (12001,)),                                   # adapter trimming
    "bc_e1": ("atac", {}, "pe", (1, False), (12001, 131072)),
    "bc_e2": ("atac", {}, "pe", (2, False), (4999,)),
    "bc_e1_notinwl": ("atac", {}, "pe", (1, True), (12001,)),
    "se_n3": ("", dict(max_num_best_mappings=3, mapq_threshold=0), "se", None, (12001,)),
    "se_bc": ("atac", {}, "se", (1, False), (4999,)),
    "hic": ("hic", dict(mapq_threshold=0), "hic", None, (12001,)),                 # split alignment, pairs records
    "sam_pe": ("", dict(mapq_threshold=0, max_num_best_mappings=2), "sam_pe", None, (4999,)),   # cmx_map_batch_pe with output_format 4
    "sam_se": ("", dict(mapq_threshold=0, max_num_best_mappings=2), "sam_se", None, (4999,)),
}


def n_pairs_for(bs):
    """At least 3 whole batches and a partial last one: 4 batches (1 + 1 + 2 over 3 lanes), or 5 for 4,999.  The last
    batch of the 12,001 runs (10,500 pairs) still has two taskloop chunks, of 5,250 each (no remainder); 131,072: 4 batches,
    the last of 40,000 pairs."""
    return {12001: 3 * 12001 + 10500, 4999: 4 * 4999 + 2000, 131072: 3 * 131072 + 40000}[bs]


def _in_batches(n, bs):
    return [(b0, min(n, b0 + bs)) for b0 in range(0, n, bs)]


def _chunk_starts(n, bs):
    """The first pair of every taskloop chunk of every batch but the call's first."""
    return [b0 + s for b0, b1 in _in_batches(n, bs) for s in cb.taskloop_chunks(b1 - b0)][1:]


def _slice(s, o, b0, b1):
    return s[o[b0]:o[b1]], (o[b0:b1 + 1] - o[b0]).astype(np.uint32)


def _oracle_batch(kind, op, bc, oidx, oref, reads, b0, b1, n_threads):
    """One oracle call over pairs [b0, b1): (records, barcode keys | None, [in whitelist, corrected] | None, trace | None)."""
    s1, o1, s2, o2 = reads["pairs"]
    a1, c1 = _slice(s1, o1, b0, b1)
    a2, c2 = _slice(s2, o2, b0, b1)
    rid = BASE + b0
    if kind in ("sam_pe", "sam_se"):
        pe = kind == "sam_pe"
        return orc.map_sam_cores(op, oidx, oref, a1, c1, a2 if pe else None, c2 if pe else None, first_read_id=rid), None, None, None
    if bc is None:
        if kind == "se":
            return orc.map_reads_se(op, oidx, oref, a1, c1, first_read_id=rid, n_threads=n_threads), None, None, None
        recs, tr = orc.map_pairs(op, oidx, oref, a1, c1, a2, c2, first_read_id=rid, n_threads=n_threads, trace=True)
        return recs, None, None, tr
    err, out_nw = bc
    L = orc.lib()
    m = L.orc_mapper_create(C.byref(op), oidx.h, oref.h)
    L.orc_mapper_set_barcodes(m, reads["wl"].h, err, 0.9, int(out_nw))
    bl = reads["bc_len"]
    bs_, bq = reads["bcs"][b0 * bl:b1 * bl], reads["quals"][b0 * bl:b1 * bl]
    n = b1 - b0
    out = np.zeros(n * op.max_num_best_mappings, dtype=orc.PE_RECORD)
    obc = np.zeros(len(out), dtype=np.uint64)
    st = np.zeros(2, dtype=np.uint64)
    if kind == "se":
        got = L.orc_map_reads_se_bc(m, n, a1.ctypes.data, c1.ctypes.data, bs_.ctypes.data, bq.ctypes.data, bl, rid, out.ctypes.data, obc.ctypes.data,
                                    len(out), n_threads, st.ctypes.data)
    else:
        got = L.orc_map_pairs_bc(m, n, a1.ctypes.data, c1.ctypes.data, a2.ctypes.data, c2.ctypes.data, bs_.ctypes.data, bq.ctypes.data, bl, rid,
                                 out.ctypes.data, obc.ctypes.data, len(out), n_threads, st.ctypes.data)
    L.orc_mapper_free(m)
    tr = None
    if kind == "pe":  # the pair's mapping does not depend on its barcode: the trace of the same pairs without barcodes
        _, tr = orc.map_pairs(op, oidx, oref, a1, c1, a2, c2, first_read_id=rid, n_threads=n_threads, trace=True)
    return out[:got], obc[:got], st, tr


def oracle_run(kind, op, bc, reads, bs):
    """The oracle over the call, one call per reference batch (batches in parallel; each call is deterministic whatever its
    thread count), concatenated."""
    oref, oidx = oracle_index()
    n = len(reads["pairs"][1]) - 1
    batches = _in_batches(n, bs)
    workers = min(len(batches), CPUS)
    with ThreadPoolExecutor(workers) as ex:
        parts = list(ex.map(lambda b: _oracle_batch(kind, op, bc, oidx, oref, reads, b[0], b[1], max(1, CPUS // workers)), batches))
    recs = np.concatenate([p[0] for p in parts])
    keys = np.concatenate([p[1] for p in parts]) if bc else None
    st = [p[2] for p in parts] if bc else None
    tr = np.concatenate([p[3] for p in parts]) if parts[0][3] is not None else None
    return recs, keys, st, tr


@functools.lru_cache(maxsize=None)
def inputs(hic, bs, barcoded, tmp):
    n = n_pairs_for(bs)
    reads = dict(pairs=make_reads(n, seed=bs + (7 if hic else 0), hic=hic, length=150 if hic else None, in_segment=_chunk_starts(n, bs)))
    if barcoded:
        path = os.path.join(tmp, "wl_%d.txt" % bs)
        bcs, quals, bl = make_barcodes(n, bs + 1, path)
        wl = orc.Whitelist(path, bl)
        wl.sample(bcs)
        reads.update(bcs=bcs, quals=quals, bc_len=bl, wl=wl)
    return reads


def _mapper(preset, kw, kind, bc, bs, reads):
    seqs, _ = reference()
    extra = dict(single_end=1) if kind in ("se", "sam_se") else {}
    if kind.startswith("sam"):
        extra["output_format"] = 4  # the oracle's SAM cores come from its BED parameters
    mrl = 75 if kind == "hic" else 64  # 2x150 Hi-C: every read in tier 1; the others: 100 bases in tier 1, 150 in tier 2
    m = cb.Mapper(cb.make_params(preset, max_read_length=mrl, batch_size=bs, **kw, **extra))
    m.upload_reference(seqs, ["chr%d" % (i + 1) for i in range(N_SEQ)])
    a = oracle_index()[1].arrays()
    m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    if bc:
        keys, counts, ns = reads["wl"].arrays()
        m.upload_barcode_whitelist(keys, counts, ns, reads["bc_len"], err_threshold=bc[0], prob_threshold=0.9, output_not_in_whitelist=bc[1])
    return m


def map_call(m, reads, single_end, on_device, lanes):
    """cmx_map_batch_pe over the whole call: host buffers into host records, or device buffers into device records (barcode
    keys always come back to the host).  Returns (records, barcode keys | None, counters, timing)."""
    import torch
    m.set_lanes(lanes)
    s1, o1, s2, o2 = reads["pairs"]
    n = len(o1) - 1
    bc = "bcs" in reads
    dt = cb.SAM_RECORD if m.params.output_format == 4 else cb.PAIRS_RECORD if m.params.output_format == 5 else cb.PE_RECORD
    cap = n * m.params.max_num_best_mappings
    keep = []

    def ptr(a):
        if a is None:
            return None
        if on_device:
            t = torch.from_numpy(a.view(np.uint8) if a.dtype == np.uint8 else a.view(np.int32)).cuda()
            keep.append(t)
            return t.data_ptr()
        return a.ctypes.data
    b = Batch(n, ptr(s1), ptr(o1), None if single_end else ptr(s2), None if single_end else ptr(o2), BASE, 1 if on_device else 0,
              ptr(reads["bcs"]) if bc else None, ptr(reads["quals"]) if bc else None, reads["bc_len"] if bc else 0)
    if on_device:
        out = torch.zeros(cap * dt.itemsize, dtype=torch.uint8, device="cuda")
        out_ptr = out.data_ptr()
    else:
        out = np.zeros(cap, dtype=dt)
        out_ptr = out.ctypes.data
    bck = np.zeros(cap, dtype=np.uint64) if bc else None
    r = Records(out_ptr, cap, 0, 1 if on_device else 0, 0, 0, 0, 0, bck.ctypes.data if bc else None, 0, 0)
    m._check(m.L.cmx_map_batch_pe(m.h, C.byref(b), C.byref(r), None), "cmx_map_batch_pe")
    k = r.n_records
    recs = out[:k * dt.itemsize].cpu().numpy().view(dt) if on_device else out[:k]
    counters = dict(n_records=k, n_mapped_pairs=r.n_mapped_pairs, n_uniquely_mapped_pairs=r.n_uniquely_mapped_pairs, n_candidates=r.n_candidates,
                    n_overflow_pairs=r.n_overflow_pairs, n_barcodes_in_whitelist=r.n_barcodes_in_whitelist, n_barcodes_corrected=r.n_barcodes_corrected)
    return recs, (bck[:k] if bc else None), counters, m.timing()


def assert_same_records(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in want.dtype.names:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def assert_same_sam(got, want, paired, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("read_id", "rid", "mapq", "is_unique", "secondary", "overflow"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, (what, f, bad[:5])
    for q in range(2 if paired else 1):
        for f in ("pos", "end", "strand", "n_cigar"):
            bad = np.nonzero(got[f][:, q] != want[f][:, q])[0]
            assert len(bad) == 0, (what, f, q, bad[:5], got[f][bad[:5], q], want[f][bad[:5], q])
        used = np.arange(want["cigar"].shape[2])[None, :] < want["n_cigar"][:, q, None]
        bad = np.nonzero(((got["cigar"][:, q] != want["cigar"][:, q]) & used).any(axis=1))[0]
        assert len(bad) == 0, (what, "cigar", q, bad[:5])


def _raw_keys(bcs, bc_len):
    """2 bits per base, first base in the high bits; rows with an N are marked by -1."""
    b = bcs.reshape(-1, bc_len)
    code = np.searchsorted(ACGT, b).astype(np.uint64)
    keys = (code << (2 * np.arange(bc_len - 1, -1, -1, dtype=np.uint64))[None, :]).sum(axis=1, dtype=np.uint64)
    keys[(b == ord("N")).any(axis=1)] = np.uint64(0xFFFFFFFFFFFFFFFF)
    return keys


def _lane_ranges(n, bs, lanes):
    n_sub = (n + bs - 1) // bs
    nl = min(lanes, n_sub)
    return [(n_sub * l // nl * bs, min(n, n_sub * (l + 1) // nl * bs)) for l in range(nl)]


CASES = [(name, bs) for name in CONFIGS for bs in CONFIGS[name][4]]


@pytest.mark.parametrize("name,bs", CASES, ids=["%s-bs%d" % c for c in CASES])
def test_call_across_batches_and_lanes_equals_per_batch_oracle(name, bs, tmp_path_factory):
    preset, kw, kind, bc, _ = CONFIGS[name]
    tmp = str(tmp_path_factory.getbasetemp())
    reads = inputs(kind == "hic", bs, bc is not None, tmp)
    n = len(reads["pairs"][1]) - 1
    n_batches = (n + bs - 1) // bs
    assert n_batches >= 4
    extra = dict(single_end=1) if kind in ("se", "sam_se") else {}
    op = orc.make_params(preset, **kw, **extra)
    want, want_keys, want_st, tr = oracle_run(kind, op, bc, reads, bs)
    assert len(want) > n // 4, len(want)
    rid0 = want["read_id"]
    assert rid0.min() >= BASE and rid0.max() < BASE + n
    single_end = kind in ("se", "sam_se")
    m = _mapper(preset, kw, kind, bc, bs, reads)
    try:
        runs = {}
        for on_device in (False, True):
            for lanes in (1, 3, 4):
                what = "%s bs=%d lanes=%d %s" % (name, bs, lanes, "device" if on_device else "host")
                recs, keys, counters, tm = map_call(m, reads, single_end, on_device, lanes)
                if kind.startswith("sam"):
                    assert_same_sam(recs, want, kind == "sam_pe", what)
                else:
                    assert_same_records(recs, want, what)
                if bc:
                    assert np.array_equal(keys, want_keys), what
                    tot = np.sum(want_st, axis=0)
                    assert (counters["n_barcodes_in_whitelist"], counters["n_barcodes_corrected"]) == (int(tot[0]), int(tot[1])), what
                assert counters["n_overflow_pairs"] == 0, what
                assert tm["tier_pairs"][1] > 0 and (kind == "hic" or tm["tier_pairs"][2] > 0), (what, list(tm["tier_pairs"]))
                runs[what] = counters
        first = next(iter(runs.values()))
        for what, c in runs.items():  # the results do not depend on the lane count or where the buffers live
            assert c == first, (what, c, first)
    finally:
        m.close()
    # floors
    if tr is not None and bs == 12001:
        mb = op.max_num_best_mappings
        sampled = np.flatnonzero(tr["n_best_pairs"] > mb)
        bounds = _chunk_starts(n, bs)
        assert len(bounds) >= 7
        for b in bounds:  # the first pair of a chunk is sampled: a start one pair off gives it another generator state
            assert b in sampled and ((sampled >= b - 200) & (sampled < b)).any() and ((sampled > b) & (sampled < b + 200)).any(), (name, b)
    if bc:
        raw = _raw_keys(reads["bcs"], reads["bc_len"])
        i = want["read_id"].astype(np.int64) - BASE
        corrected = (raw[i] != want_keys) & (raw[i] != np.uint64(0xFFFFFFFFFFFFFFFF))
        for lo, hi in _lane_ranges(n, bs, 4) + _lane_ranges(n, bs, 3):
            assert (corrected & (i >= lo) & (i < hi)).any(), (name, lo, hi)
