"""ctypes binding of include/chromap_b200.h.  Mirrors the reference's paired-end mapping call
(Chromap::MapPairedEndReads, chromap.h:636) at batch granularity."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path():
    return os.path.join(_HERE, "libchromap_b200.so")


class CmxError(RuntimeError):
    pass


class Params(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "error_threshold", "min_num_seeds", "max_seed_freq0", "max_seed_freq1", "max_num_best_mappings",
        "max_insert_size", "mapq_threshold", "min_read_length", "drop_repetitive_reads", "trim_adapters",
        "remove_pcr_duplicates", "tn5_shift", "split_alignment", "low_memory_mode", "output_format",
        "batch_size", "max_read_length", "single_end")]


SAM_RECORD = np.dtype([("read_id", "<u4"), ("rid", "<u4"), ("pos", "<u4", 2), ("end", "<u4", 2), ("strand", "u1", 2), ("mapq", "u1"), ("is_unique", "u1"),
                       ("secondary", "u1"), ("n_cigar", "u1", 2), ("overflow", "u1"), ("cigar", "<u4", (2, 24))], align=True)


class ReadSet(C.Structure):
    _fields_ = [("names", C.c_void_p), ("seq", C.c_void_p), ("off", C.c_void_p), ("qual", C.c_void_p)]


def _sam_read_set(r, keep):
    """cmx_read_set of (names, seqs, quals) lists of bytes (quals may be None); keep holds the buffers alive."""
    if r is None:
        return None
    nm, sq, ql = r
    arr = (C.c_char_p * len(nm))(*nm)
    seq = np.frombuffer(b"".join(sq), dtype=np.uint8)
    off = np.zeros(len(sq) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in sq])
    qual = np.frombuffer(b"".join(ql), dtype=np.uint8) if ql is not None else None
    keep.extend([arr, seq, off, qual])
    return ReadSet(C.cast(arr, C.c_void_p), seq.ctypes.data, off.ctypes.data, qual.ctypes.data if qual is not None else None)


def format_sam(params, ref_names, ref_seqs, records, reads1, reads2=None, first_read_id=0):
    """SAM text from SAM cores (host only).  ref_seqs: list of uint8 arrays; reads*: (names, seqs, quals) lists of bytes."""
    return _format_sam_host("cmx_format_sam", params, ref_names, ref_seqs, records, None, 0, reads1, reads2, first_read_id, None)


def format_sam_bc(params, ref_names, ref_seqs, records, bcs, bc_len, reads1, reads2=None, first_read_id=0, translation=None):
    """The same with cell barcodes (host only, cmx_format_sam_bc): bcs = one key per core (None: bulk), translation a
    BarcodeTranslation or None.  Raises BarcodeNotTranslated, CmxError for the writer's other failures."""
    return _format_sam_host("cmx_format_sam_bc", params, ref_names, ref_seqs, records, bcs, bc_len, reads1, reads2, first_read_id, translation)


def _format_sam_host(fn, params, ref_names, ref_seqs, records, bcs, bc_len, reads1, reads2, first_read_id, translation):
    L = load_library()
    names = (C.c_char_p * len(ref_names))(*[s.encode() if isinstance(s, str) else s for s in ref_names])
    lens = np.array([len(s) for s in ref_seqs], dtype=np.uint32)
    concat = np.concatenate(ref_seqs).astype(np.uint8)
    roff = np.zeros(len(ref_seqs) + 1, dtype=np.uint64)
    roff[1:] = np.cumsum(lens.astype(np.uint64))
    keep = []
    r1, r2 = _sam_read_set(reads1, keep), _sam_read_set(reads2, keep)
    recs = np.ascontiguousarray(records)
    head = (C.byref(params), names, lens.ctypes.data, len(ref_names), concat.ctypes.data, roff.ctypes.data, recs.ctypes.data)
    reads = (C.byref(r1), C.byref(r2) if r2 is not None else None, first_read_id)
    if fn == "cmx_format_sam":
        args = head + (len(recs),) + reads
    else:
        bp = np.ascontiguousarray(bcs, dtype=np.uint64) if bcs is not None else None
        t = translation.struct() if translation is not None else None
        keep.extend([bp, t])
        args = head + (bp.ctypes.data if bp is not None else None, bc_len, len(recs)) + reads + (C.byref(t) if t is not None else None,)
    f = getattr(L, fn)
    n = f(*args, None, 0)
    if n == ERR_BARCODE_TRANSLATE:
        raise BarcodeNotTranslated("Barcode does not exist in the translation table.")
    if n < 0:
        raise CmxError("%s failed (%d)" % (fn, n))
    buf = C.create_string_buffer(n + 1)
    assert f(*args, buf, n) == n
    return buf.raw[:n]


def format_paf(params, ref_names, ref_lengths, records, names1, lengths1, names2=None, lengths2=None, first_read_id=0):
    """PAF text from BED-path records as map_batch returned them (host only; orders / dedups / filters itself)."""
    L = load_library()
    rn = (C.c_char_p * len(ref_names))(*[s.encode() if isinstance(s, str) else s for s in ref_names])
    rl = np.ascontiguousarray(ref_lengths, dtype=np.uint32)
    n1 = (C.c_char_p * len(names1))(*names1)
    l1 = np.ascontiguousarray(lengths1, dtype=np.uint16)
    n2 = (C.c_char_p * len(names2))(*names2) if names2 is not None else None
    l2 = np.ascontiguousarray(lengths2, dtype=np.uint16) if lengths2 is not None else None
    recs = np.ascontiguousarray(records)
    args = (C.byref(params), rn, rl.ctypes.data, recs.ctypes.data, len(recs), n1, l1.ctypes.data, n2, l2.ctypes.data if l2 is not None else None, first_read_id)
    n = L.cmx_format_paf(*args, None, 0)
    if n < 0:
        raise CmxError("cmx_format_paf failed (%d)" % n)
    buf = C.create_string_buffer(n + 1)
    assert L.cmx_format_paf(*args, buf, n) == n
    return buf.raw[:n]


class Ingested(C.Structure):
    _fields_ = [("n_reads", C.c_uint32), ("seq", C.c_void_p), ("off", C.c_void_p), ("qual", C.c_void_p), ("min_len", C.c_uint32), ("max_len", C.c_uint32)]


MAX_READ_RANGES = 8


class ReadRange(C.Structure):
    """cmx_read_range: the part of every read of one file that --read-format keeps."""
    _fields_ = [("n", C.c_uint32), ("start", C.c_int32 * MAX_READ_RANGES), ("end", C.c_int32 * MAX_READ_RANGES), ("reverse", C.c_int32)]

    def ranges(self):
        return [(self.start[k], self.end[k]) for k in range(self.n)]


def parse_read_format(fmt):
    """--read-format text -> (r1, r2, bc) ReadRange (host only).  Raises CmxError for a format outside the grammar and for
    ranges the GPU path refuses (not ascending and disjoint, -1 before the last range, more than 8 per file)."""
    L = load_library()
    r = [ReadRange() for _ in range(3)]
    rc = L.cmx_parse_read_format(fmt.encode() if isinstance(fmt, str) else fmt, *[C.byref(x) for x in r])
    if rc == -3:
        raise CmxError("Unknown read format: %s" % fmt)
    if rc != 0:
        raise CmxError("read format %s: ranges the GPU path refuses (%d)" % (fmt, rc))
    return tuple(r)


def apply_read_range(read_range, seq, qual=None):
    """The cut of one read (host only): (seq, qual) bytes after it.  Raises CmxError when an explicit end is at or past the
    read's length or nothing is left."""
    L = load_library()
    s = C.create_string_buffer(bytes(seq), len(seq))
    q = C.create_string_buffer(bytes(qual), len(qual)) if qual is not None else None
    n = L.cmx_apply_read_range(C.byref(read_range), s, q, len(seq))
    if n <= 0:
        raise CmxError("read of length %d: %s" % (len(seq), "empty after the cut" if n == 0 else "shorter than a range's end (%d)" % n))
    return s.raw[:n], (q.raw[:n] if q is not None else None)


class _Translation(C.Structure):
    _fields_ = [("n", C.c_uint64), ("keys", C.c_void_p), ("to_off", C.c_void_p), ("to", C.c_void_p), ("from_len", C.c_uint32)]


ERR_BARCODE_TRANSLATE = -8  # CMX_ERR_BARCODE_TRANSLATE


class BarcodeNotTranslated(CmxError):
    """A barcode segment has no entry in the --barcode-translate table (CMX_ERR_BARCODE_TRANSLATE)."""


class BarcodeTranslation:
    """A --barcode-translate table: distinct FROM keys (2 bits per base), the TO string of each (bytes) and the FROM length L."""

    def __init__(self, keys, to, from_len):
        self.keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self.to = [bytes(t) for t in to]
        self.from_len = int(from_len)
        assert len(self.keys) == len(self.to)
        self._off = np.zeros(len(self.to) + 1, dtype=np.uint64)
        self._off[1:] = np.cumsum([len(t) for t in self.to], dtype=np.uint64)
        self._blob = C.create_string_buffer(b"".join(self.to), int(self._off[-1]) + 1)

    def struct(self):
        """The cmx_barcode_translation view (valid while this object lives)."""
        return _Translation(len(self.keys), self.keys.ctypes.data, self._off.ctypes.data, C.addressof(self._blob), self.from_len)


def parse_barcode_translation(data):
    """Bytes of a --barcode-translate file (already inflated) -> BarcodeTranslation (host only).  Raises CmxError, naming the
    line, for a table the GPU path refuses."""
    L = load_library()
    data = bytes(data)
    t, err = _Translation(), C.create_string_buffer(256)
    rc = L.cmx_parse_barcode_translation(data, len(data), C.byref(t), err, len(err))
    if rc != 0:
        raise CmxError("barcode translation table refused: " + err.value.decode())
    try:
        off = np.ctypeslib.as_array(C.cast(t.to_off, C.POINTER(C.c_uint64)), (t.n + 1,)).copy()
        keys = np.ctypeslib.as_array(C.cast(t.keys, C.POINTER(C.c_uint64)), (t.n,)).copy()
        blob = C.string_at(t.to, int(off[-1])) if off[-1] else b""
        return BarcodeTranslation(keys, [blob[off[i]:off[i + 1]] for i in range(t.n)], t.from_len)
    finally:
        L.cmx_free_barcode_translation(C.byref(t))


def format_bed_bc_tr(names, recs, bcs, bc_len, translation):
    """Barcoded BED text on the host with a BarcodeTranslation applied (None: the untranslated text), the twin of
    Mapper.format_bed_gpu with an uploaded table.  Raises BarcodeNotTranslated."""
    L = load_library()
    arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
    recs = np.ascontiguousarray(recs); bcs = np.ascontiguousarray(bcs, dtype=np.uint64)
    t = translation.struct() if translation is not None else None
    args = (arr, recs.ctypes.data, bcs.ctypes.data, len(recs), bc_len, C.byref(t) if t is not None else None)
    n = L.cmx_format_bed_bc_tr(*args, None, 0)
    if n == -8:
        raise BarcodeNotTranslated("Barcode does not exist in the translation table.")
    if n < 0:
        raise CmxError("cmx_format_bed_bc_tr failed (%d)" % n)
    buf = C.create_string_buffer(n + 1)
    assert L.cmx_format_bed_bc_tr(*args, buf, n) == n
    return buf.raw[:n]


class BulkDedupError(CmxError):
    """A bulk-level duplicate removal refused: its status in `.status` (records untouched)."""

    def __init__(self, msg, status):
        super().__init__(msg)
        self.status = status


def postprocess_bc_bulk(params, wl_keys, wl_counts, recs, bcs):
    """Host twin of Mapper.postprocess_bc_bulk_gpu (the reference's low-memory merge loop at bulk level), with the whitelist
    given as keys and their counts.  Returns (records, barcode keys); raises BulkDedupError."""
    L = load_library()
    recs = np.ascontiguousarray(recs.copy()); bcs = np.ascontiguousarray(np.array(bcs, dtype=np.uint64).copy())
    wk = np.ascontiguousarray(wl_keys, dtype=np.uint64); wc = np.ascontiguousarray(wl_counts, dtype=np.uint32)
    n = C.c_uint64()
    rc = L.cmx_postprocess_bc_bulk(C.byref(params), wk.ctypes.data, wc.ctypes.data, len(wk), recs.ctypes.data, bcs.ctypes.data, len(recs), C.byref(n))
    if rc != 0:
        raise BulkDedupError("cmx_postprocess_bc_bulk failed (%d)" % rc, rc)
    return recs[:n.value], bcs[:n.value]


class Batch(C.Structure):
    _fields_ = [("n_pairs", C.c_uint32), ("seq1", C.c_void_p), ("off1", C.c_void_p), ("seq2", C.c_void_p),
                ("off2", C.c_void_p), ("first_read_id", C.c_uint32), ("on_device", C.c_int32),
                ("bc_seq", C.c_void_p), ("bc_qual", C.c_void_p), ("bc_len", C.c_uint32)]


class Records(C.Structure):
    _fields_ = [("records", C.c_void_p), ("capacity", C.c_uint64), ("n_records", C.c_uint64), ("on_device", C.c_int32),
                ("n_mapped_pairs", C.c_uint64), ("n_uniquely_mapped_pairs", C.c_uint64), ("n_candidates", C.c_uint64),
                ("n_overflow_pairs", C.c_uint64), ("barcode_keys", C.c_void_p), ("n_barcodes_in_whitelist", C.c_uint64),
                ("n_barcodes_corrected", C.c_uint64)]


class Timing(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("h2d_ms", "seed_ms", "pair_candidates_ms", "verify_ms", "pairing_ms",
                                         "select_ms", "emit_ms", "d2h_ms", "total_ms", "front_ms", "reserved_ms", "cluster_ms")] + \
               [(n, C.c_uint64) for n in ("n_minimizers", "n_probe_steps", "n_found", "n_occ_reads", "n_verified",
                                          "n_launches")] + [("tier_pairs", C.c_uint64 * 3), ("escalations", C.c_uint64 * 8)]

    def asdict(self):
        d = {n: getattr(self, n) for n, _ in self._fields_}
        d["tier_pairs"] = list(d["tier_pairs"]); d["escalations"] = list(d["escalations"])
        return d


class ExchangeStats(C.Structure):
    _fields_ = [("pack_ms", C.c_float), ("allgather_ms", C.c_float), ("resolve_ms", C.c_float), ("bytes_sent", C.c_uint64),
                ("bytes_received", C.c_uint64), ("n_global", C.c_uint64), ("n_ranks", C.c_uint32), ("pad", C.c_uint32)]

    def asdict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "pad"}


class ShuffleStats(C.Structure):
    _fields_ = [("partition_ms", C.c_float), ("shuffle_ms", C.c_float), ("postprocess_ms", C.c_float), ("n_ranks", C.c_uint32),
                ("bytes_sent", C.c_uint64), ("bytes_received", C.c_uint64), ("n_received", C.c_uint64), ("n_global", C.c_uint64)]

    def asdict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


PE_RECORD = np.dtype([("read_id", "<u4"), ("rid", "<u4"), ("fragment_start", "<u4"), ("fragment_length", "<u2"),
                      ("mapq", "u1"), ("direction", "u1"), ("is_unique", "u1"), ("num_dups", "u1"),
                      ("positive_alignment_length", "<u2"), ("negative_alignment_length", "<u2")], align=True)
assert PE_RECORD.itemsize == 24

PAIRS_RECORD = np.dtype([("read_id", "<u4"), ("rid1", "<u4"), ("rid2", "<u4"), ("pos1", "<u4"), ("pos2", "<u4"), ("strand1", "u1"),
                         ("strand2", "u1"), ("mapq", "u1"), ("is_unique", "u1")], align=True)
assert PAIRS_RECORD.itemsize == 24

PAIR_TRACE = np.dtype([("n_minimizers", "<i4", 2), ("n_pos_candidates_gen", "<i4", 2), ("n_neg_candidates_gen", "<i4", 2),
                       ("n_pos_candidates", "<i4", 2), ("n_neg_candidates", "<i4", 2), ("n_pos_mappings", "<i4", 2),
                       ("n_neg_mappings", "<i4", 2), ("min_errors", "<i4", 2), ("second_min_errors", "<i4", 2),
                       ("n_best", "<i4", 2), ("n_second_best", "<i4", 2), ("repetitive_seed_length", "<u4", 2),
                       ("supplement_result", "<i4"), ("min_sum_errors", "<i4"), ("second_min_sum_errors", "<i4"),
                       ("n_best_pairs", "<i4"), ("n_second_best_pairs", "<i4"), ("n_records", "<i4"),
                       ("trimmed_len", "<i4", 2)], align=True)

_lib = None


class AllocationStats(C.Structure):  # cmx_allocation_stats
    _fields_ = [(n, C.c_uint64) for n in ("n_multi", "n_allocated", "n_without_overlap", "n_draws", "n_uni_after", "n_multi_after")]


def load_library():
    """Load the CUDA C-ABI library.  Fails loudly when it has not been built — there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise CmxError("chromap_b200: %s is missing — run __graft_entry__.build() (nvcc, sm_90a). "
                       "There is no CPU fallback." % p)
    L = C.CDLL(p)
    vp, u32, u64, i32, i64 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_int64
    L.cmx_default_params.argtypes = [C.POINTER(Params)]
    L.cmx_apply_preset.argtypes = [C.POINTER(Params), C.c_char_p]
    L.cmx_create.argtypes = [C.POINTER(vp), i32, C.POINTER(Params)]
    L.cmx_destroy.argtypes = [vp]
    L.cmx_last_error.restype = C.c_char_p; L.cmx_last_error.argtypes = [vp]
    L.cmx_upload_reference.argtypes = [vp, u32, vp, vp]
    L.cmx_upload_index.argtypes = [vp, i32, i32, u32, vp, vp, vp, vp, u32]
    L.cmx_build_index.argtypes = [vp, i32, i32]
    L.cmx_download_index.argtypes = [vp, C.POINTER(u32), C.POINTER(u32), vp, vp, vp, C.POINTER(u32), vp]
    L.cmx_index_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.cmx_map_batch_pe.argtypes = [vp, C.POINTER(Batch), C.POINTER(Records), vp]
    L.cmx_upload_barcode_whitelist.argtypes = [vp, vp, vp, u64, u64, u32, i32, C.c_double, i32]
    L.cmx_postprocess_bc.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    L.cmx_format_bed_bc.restype = i64; L.cmx_format_bed_bc.argtypes = [vp, vp, vp, u64, u32, vp, i64]
    L.cmx_postprocess.argtypes = [vp, vp, u64, C.POINTER(u64)]
    L.cmx_format_bed.restype = i64; L.cmx_format_bed.argtypes = [vp, vp, u64, vp, i64]
    L.cmx_format_tagalign.restype = i64; L.cmx_format_tagalign.argtypes = [vp, vp, u64, vp, i64]
    L.cmx_format_pairs_gpu.restype = i64; L.cmx_format_pairs_gpu.argtypes = [vp, vp, vp, u32, vp, u64, vp, u64, u32, vp, i64]
    L.cmx_format_bed_gpu.restype = i64; L.cmx_format_bed_gpu.argtypes = [vp, vp, vp, vp, u64, u32, vp, i64]
    L.cmx_postprocess_pairs.argtypes = [vp, vp, u64, C.POINTER(u64)]
    L.cmx_postprocess_gpu.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    L.cmx_format_pairs.restype = i64; L.cmx_format_pairs.argtypes = [vp, vp, u32, vp, u64, vp, u32, vp, i64]
    L.cmx_stage_minimizers.argtypes = [vp, C.POINTER(Batch), vp, vp, vp, u32]
    L.cmx_stage_probe.argtypes = [vp, vp, u64, vp, vp, vp]
    L.cmx_stage_banded_align.argtypes = [vp, i32, i32, vp, vp, u64, vp, vp]
    L.cmx_stage_cta_sort.argtypes = [vp, vp, vp, u32, u32]
    L.cmx_stage_correct_barcodes.argtypes = [vp, vp, vp, u64, u32, vp, vp, vp, vp]
    L.cmx_last_batch_trace.argtypes = [vp, vp, u32]
    L.cmx_last_batch_timing.argtypes = [vp, C.POINTER(Timing)]
    L.cmx_set_lanes.argtypes = [vp, i32]
    L.cmx_set_max_read_length.argtypes = [vp, i32]
    L.cmx_host_register.argtypes = [vp, u64]
    L.cmx_host_unregister.argtypes = [vp]
    L.cmx_format_paf.restype = i64
    L.cmx_format_paf.argtypes = [C.POINTER(Params), vp, vp, vp, u64, vp, vp, vp, vp, u32, vp, i64]
    L.cmx_format_sam.restype = i64
    L.cmx_format_sam.argtypes = [C.POINTER(Params), vp, vp, u32, vp, vp, vp, u64, C.POINTER(ReadSet), C.POINTER(ReadSet), u32, vp, i64]
    L.cmx_format_sam_bc.restype = i64
    L.cmx_format_sam_bc.argtypes = [C.POINTER(Params), vp, vp, u32, vp, vp, vp, vp, u32, u64, C.POINTER(ReadSet), C.POINTER(ReadSet), u32,
                                    C.POINTER(_Translation), vp, i64]
    L.cmx_format_sam_gpu.restype = i64
    L.cmx_format_sam_gpu.argtypes = [vp, vp, vp, u32, vp, vp, u32, u64, C.POINTER(ReadSet), C.POINTER(ReadSet), u32, vp, i64]
    L.cmx_comm_unique_id.argtypes = [vp]
    L.cmx_comm_init.argtypes = [vp, i32, i32, vp]
    L.cmx_comm_destroy.argtypes = [vp]
    L.cmx_dedup_exchange.argtypes = [vp, vp, vp, u64, i32, vp, vp, C.POINTER(u64), C.POINTER(ExchangeStats)]
    L.cmx_dedup_shuffle.argtypes = [vp, vp, vp, u64, i32, vp, vp, u64, C.POINTER(u64), C.POINTER(ShuffleStats)]
    L.cmx_exchange_finish.argtypes = [C.POINTER(Params), vp, vp, u64]
    L.cmx_fastq_cut.restype = u64; L.cmx_fastq_cut.argtypes = [vp, u64, u32, C.POINTER(u32)]
    L.cmx_ingest_fastq.argtypes = [vp, i32, vp, u64, i32, vp, C.POINTER(Ingested)]
    L.cmx_parse_read_format.argtypes = [C.c_char_p, C.POINTER(ReadRange), C.POINTER(ReadRange), C.POINTER(ReadRange)]
    L.cmx_apply_read_range.restype = i64; L.cmx_apply_read_range.argtypes = [C.POINTER(ReadRange), vp, vp, u32]
    L.cmx_parse_barcode_translation.argtypes = [C.c_char_p, u64, C.POINTER(_Translation), vp, u64]
    L.cmx_free_barcode_translation.restype = None; L.cmx_free_barcode_translation.argtypes = [C.POINTER(_Translation)]
    L.cmx_upload_barcode_translation.argtypes = [vp, C.POINTER(_Translation)]
    L.cmx_format_bed_bc_tr.restype = i64; L.cmx_format_bed_bc_tr.argtypes = [vp, vp, vp, u64, u32, C.POINTER(_Translation), vp, i64]
    L.cmx_ingest_fastq_range.argtypes = [vp, i32, vp, u64, i32, vp, C.POINTER(ReadRange), C.POINTER(Ingested)]
    L.cmx_postprocess_bc_bulk_gpu.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    L.cmx_postprocess_bc_bulk.argtypes = [C.POINTER(Params), vp, vp, u64, vp, vp, u64, C.POINTER(u64)]
    for f in (L.cmx_allocate_multi_mappings_gpu, L.cmx_allocate_multi_mappings):
        f.argtypes = [vp, vp, vp, u64, C.c_int32, C.c_int32, C.POINTER(u64), C.POINTER(AllocationStats)]
    _lib = L
    return L


def make_params(preset="", **kw):
    L = load_library()
    p = Params()
    L.cmx_default_params(C.byref(p))
    if L.cmx_apply_preset(C.byref(p), preset.encode()) != 0:
        raise CmxError("Unrecognized preset parameters " + preset)
    for k, v in kw.items():
        setattr(p, k, int(v))
    return p


def exchange_finish(params, recs, barcode_keys=None):
    """Reference order + deferred Tn5 shift over the survivors of all ranks (host only, mapping_writer.h:285-287)."""
    L = load_library()
    recs = np.ascontiguousarray(recs).copy()
    bcs = np.ascontiguousarray(barcode_keys, dtype=np.uint64).copy() if barcode_keys is not None else None
    rc = L.cmx_exchange_finish(C.byref(params), recs.ctypes.data if len(recs) else None, _ptr(bcs), len(recs))
    if rc != 0:
        raise CmxError("cmx_exchange_finish failed (%d)" % rc)
    return recs if bcs is None else (recs, bcs)


def taskloop_chunks(n, grain=5000):
    """Chunk starts of the reference's `taskloop grainsize(5000)` (chromap.h:892) over n pairs."""
    nt = max(1, n // grain)
    chunk, rem = divmod(n, nt)
    starts, s = [], 0
    for t in range(nt):
        starts.append(s)
        s += chunk + (1 if t < rem else 0)
    return starts


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):  # torch tensor
        return a.data_ptr()
    return int(a)


class Mapper:
    """One GPU context: reference + index resident in HBM, batches of read pairs in, PE records out."""

    def __init__(self, params=None, device=0):
        self.L = load_library()
        self.params = params if params is not None else make_params()
        h = C.c_void_p()
        rc = self.L.cmx_create(C.byref(h), device, C.byref(self.params))
        if rc == -1:
            raise CmxError("chromap_b200: no CUDA device — the product path has no CPU fallback")
        if rc != 0:
            raise CmxError("cmx_create failed (%d): unsupported parameters" % rc)
        self.h = h
        self.names = None

    def close(self):
        if getattr(self, "h", None):
            self.L.cmx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise CmxError("%s failed (%d): %s" % (what, rc, self.L.cmx_last_error(self.h).decode()))

    def upload_reference(self, seqs, names=None):
        """seqs: list of uint8 arrays (ASCII bases as loaded)."""
        concat = np.ascontiguousarray(np.concatenate(seqs).astype(np.uint8))
        offs = np.zeros(len(seqs) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(s) for s in seqs])
        self._check(self.L.cmx_upload_reference(self.h, len(seqs), offs.ctypes.data, concat.ctypes.data), "cmx_upload_reference")
        self.names = names or ["chr%d" % (i + 1) for i in range(len(seqs))]
        self.ref_lengths = np.diff(offs).astype(np.uint32)

    def upload_reference_ptr(self, ptr, offsets, names=None):
        """Reference already concatenated in (host or device) memory at `ptr`; offsets uint64[n_seq+1]."""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        self._check(self.L.cmx_upload_reference(self.h, len(offs) - 1, offs.ctypes.data, int(ptr)), "cmx_upload_reference")
        self.names = names or ["chr%d" % (i + 1) for i in range(len(offs) - 1)]
        self.ref_lengths = np.diff(offs).astype(np.uint32)

    def upload_index(self, k, w, n_buckets, flags, keys, vals, occ):
        flags = np.ascontiguousarray(flags, dtype=np.uint32); keys = np.ascontiguousarray(keys, dtype=np.uint64)
        vals = np.ascontiguousarray(vals, dtype=np.uint64); occ = np.ascontiguousarray(occ, dtype=np.uint64)
        self._check(self.L.cmx_upload_index(self.h, k, w, n_buckets, flags.ctypes.data, keys.ctypes.data, vals.ctypes.data,
                                            occ.ctypes.data if len(occ) else None, len(occ)), "cmx_upload_index")

    def build_index(self, k=17, w=7):
        self._check(self.L.cmx_build_index(self.h, k, w), "cmx_build_index")

    def index_info(self):
        k, w = C.c_int(), C.c_int()
        nk, no, ns = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self.L.cmx_index_info(self.h, C.byref(k), C.byref(w), C.byref(nk), C.byref(no), C.byref(ns)), "cmx_index_info")
        return dict(k=k.value, w=w.value, n_keys=nk.value, n_occ=no.value, table_slots=ns.value)

    def download_index(self):
        nb, nk, no = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._check(self.L.cmx_download_index(self.h, C.byref(nb), C.byref(nk), None, None, None, C.byref(no), None), "cmx_download_index")
        flags = np.zeros(max(1, nb.value >> 4), dtype=np.uint32)
        keys = np.zeros(nb.value, dtype=np.uint64); vals = np.zeros(nb.value, dtype=np.uint64)
        occ = np.zeros(no.value, dtype=np.uint64)
        self._check(self.L.cmx_download_index(self.h, C.byref(nb), C.byref(nk), flags.ctypes.data, keys.ctypes.data, vals.ctypes.data,
                                              C.byref(no), occ.ctypes.data if no.value else None), "cmx_download_index")
        return dict(n_buckets=nb.value, n_keys=nk.value, flags=flags, keys=keys, vals=vals, occ=occ)

    def upload_barcode_whitelist(self, keys, counts, num_sample, bc_len, err_threshold=1, prob_threshold=0.9, output_not_in_whitelist=False):
        keys = np.ascontiguousarray(keys, dtype=np.uint64); counts = np.ascontiguousarray(counts, dtype=np.uint32)
        self._check(self.L.cmx_upload_barcode_whitelist(self.h, keys.ctypes.data, counts.ctypes.data, len(keys), int(num_sample), bc_len,
                                                        err_threshold, prob_threshold, int(output_not_in_whitelist)), "cmx_upload_barcode_whitelist")

    def upload_barcode_translation(self, translation):
        """Put a BarcodeTranslation on the device (None removes it): format_bed_gpu then writes translated barcode fields."""
        t = translation.struct() if translation is not None else None
        self._check(self.L.cmx_upload_barcode_translation(self.h, C.byref(t) if t is not None else None), "cmx_upload_barcode_translation")

    def map_batch(self, seq1, off1, seq2, off2, first_read_id=0, on_device=False, n_pairs=None, out=None, out_on_device=False,
                  barcodes=None, barcode_quals=None, bc_len=0):
        """Host numpy arrays (or device pointers / torch tensors when on_device).  Returns (records, stats)."""
        n = n_pairs if n_pairs is not None else len(off1) - 1
        if not on_device:
            seq1 = np.ascontiguousarray(seq1, dtype=np.uint8); off1 = np.ascontiguousarray(off1, dtype=np.uint32)
            if seq2 is not None:  # None: single-end (params.single_end)
                seq2 = np.ascontiguousarray(seq2, dtype=np.uint8); off2 = np.ascontiguousarray(off2, dtype=np.uint32)
        if barcodes is not None and not on_device:
            barcodes = np.ascontiguousarray(barcodes, dtype=np.uint8); barcode_quals = np.ascontiguousarray(barcode_quals, dtype=np.uint8)
        b = Batch(n, _ptr(seq1), _ptr(off1), _ptr(seq2), _ptr(off2), first_read_id, 1 if on_device else 0,
                  _ptr(barcodes), _ptr(barcode_quals), bc_len if barcodes is not None else 0)
        mb = self.params.max_num_best_mappings
        if out is None:
            out = np.zeros(n * mb, dtype=PAIRS_RECORD if self.params.output_format == 5 else SAM_RECORD if self.params.output_format == 4 else PE_RECORD)
        cap = (out.numel() * out.element_size() // 24) if hasattr(out, "data_ptr") else len(out)
        bck = np.zeros(cap, dtype=np.uint64) if (barcodes is not None and not out_on_device) else None
        r = Records(_ptr(out), cap, 0, 1 if out_on_device else 0, 0, 0, 0, 0, _ptr(bck), 0, 0)
        rc = self.L.cmx_map_batch_pe(self.h, C.byref(b), C.byref(r), None)
        self._check(rc, "cmx_map_batch_pe")
        stats = dict(n_records=r.n_records, n_mapped_pairs=r.n_mapped_pairs, n_uniquely_mapped_pairs=r.n_uniquely_mapped_pairs,
                     n_candidates=r.n_candidates, n_overflow_pairs=r.n_overflow_pairs, n_barcodes_in_whitelist=r.n_barcodes_in_whitelist,
                     n_barcodes_corrected=r.n_barcodes_corrected)
        if bck is not None:
            stats["barcode_keys"] = bck[:r.n_records]
        if out_on_device:
            return out, stats
        return out[:r.n_records], stats

    # ---- multi-GPU exchange (one process per GPU) ----
    @staticmethod
    def _prefer_framework_nccl():
        """When PyTorch is installed, load it (and with it its NCCL) before the library binds to one: the library takes the NCCL
        the process already holds, so both sides share a copy; without PyTorch the system libnccl.so.2 is used."""
        try:
            import torch  # noqa: F401
        except Exception:
            pass

    def comm_unique_id(self):
        self._prefer_framework_nccl()
        buf = (C.c_char * 128)()
        rc = self.L.cmx_comm_unique_id(buf)
        if rc != 0:
            raise CmxError("cmx_comm_unique_id failed (%d): NCCL not available" % rc)
        return bytes(buf)

    def comm_init(self, n_ranks, rank, unique_id):
        self._prefer_framework_nccl()
        buf = (C.c_char * 128).from_buffer_copy(unique_id)
        self._check(self.L.cmx_comm_init(self.h, n_ranks, rank, buf), "cmx_comm_init")

    def comm_destroy(self):
        self.L.cmx_comm_destroy(self.h)

    def dedup_exchange(self, recs, barcode_keys=None, on_device=False, out=None, out_bc=None, n=None):
        """This rank's records in (numpy, or device pointers / torch tensors with on_device), this rank's survivors out."""
        if on_device:
            cnt = int(n)
            no = C.c_uint64()
            st = ExchangeStats()
            self._check(self.L.cmx_dedup_exchange(self.h, _ptr(recs), _ptr(barcode_keys), cnt, 1, _ptr(out), _ptr(out_bc), C.byref(no), C.byref(st)),
                        "cmx_dedup_exchange")
            return int(no.value), st.asdict()
        recs = np.ascontiguousarray(recs)
        o = np.zeros(max(1, len(recs)), dtype=PE_RECORD)
        bcs = np.ascontiguousarray(barcode_keys, dtype=np.uint64) if barcode_keys is not None else None
        obc = np.zeros(max(1, len(recs)), dtype=np.uint64) if bcs is not None else None
        no = C.c_uint64()
        st = ExchangeStats()
        self._check(self.L.cmx_dedup_exchange(self.h, recs.ctypes.data if len(recs) else o.ctypes.data, _ptr(bcs), len(recs), 0, o.ctypes.data, _ptr(obc),
                                              C.byref(no), C.byref(st)), "cmx_dedup_exchange")
        k = int(no.value)
        if bcs is not None:
            return o[:k].copy(), obc[:k].copy(), st.asdict()
        return o[:k].copy(), st.asdict()

    def dedup_shuffle(self, recs, barcode_keys=None, on_device=False, out=None, out_bc=None, n=None, capacity=None):
        """This rank's records in; out: the records of this rank's KEY RANGE after duplicate removal over the whole run
        (reference order, num_dups set, MAPQ-filtered, Tn5 applied).  Ranks' outputs concatenated in rank order = the run's output."""
        if on_device:
            no = C.c_uint64()
            st = ShuffleStats()
            self._check(self.L.cmx_dedup_shuffle(self.h, _ptr(recs), _ptr(barcode_keys), int(n), 1, _ptr(out), _ptr(out_bc), int(capacity), C.byref(no),
                                                 C.byref(st)), "cmx_dedup_shuffle")
            return int(no.value), st.asdict()
        recs = np.ascontiguousarray(recs)
        bcs = np.ascontiguousarray(barcode_keys, dtype=np.uint64) if barcode_keys is not None else None
        cap = int(capacity) if capacity is not None else 2 * len(recs) + 4096
        while True:
            o = np.zeros(max(1, cap), dtype=PE_RECORD)
            obc = np.zeros(max(1, cap), dtype=np.uint64) if bcs is not None else None
            no = C.c_uint64()
            st = ShuffleStats()
            rc = self.L.cmx_dedup_shuffle(self.h, recs.ctypes.data if len(recs) else o.ctypes.data, _ptr(bcs), len(recs), 0, o.ctypes.data, _ptr(obc), cap,
                                          C.byref(no), C.byref(st))
            if rc != 0 and int(no.value) > cap:
                # the key range of this rank holds more than the guess.  The shuffle is collective: every rank must repeat it,
                # so the caller is told instead of retrying here on one rank only.
                raise CmxError("cmx_dedup_shuffle: capacity %d too small, %d needed" % (cap, int(no.value)))
            self._check(rc, "cmx_dedup_shuffle")
            break
        k = int(no.value)
        if bcs is not None:
            return o[:k].copy(), obc[:k].copy(), st.asdict()
        return o[:k].copy(), st.asdict()

    def fastq_cut(self, text, max_records):
        """(bytes, records) of the first min(max_records, complete) 4-line records of `text` (bytes / uint8 array)."""
        a = np.frombuffer(text, dtype=np.uint8) if not isinstance(text, np.ndarray) else text
        n = C.c_uint32()
        b = self.L.cmx_fastq_cut(a.ctypes.data, len(a), max_records, C.byref(n))
        return b, n.value

    def ingest_fastq(self, slot, text, want_qual=False, want_names=False, read_range=None):
        """FASTQ text (whole records) -> packed reads on the device, cut by read_range (a ReadRange) if given.
        Returns (Ingested, name_spans | None)."""
        a = np.frombuffer(text, dtype=np.uint8) if not isinstance(text, np.ndarray) else text
        spans = np.zeros(2 * (len(a) // 8 + 1), dtype=np.uint32) if want_names else None
        g = Ingested()
        args = (self.h, slot, a.ctypes.data, len(a), 1 if want_qual else 0, spans.ctypes.data if want_names else None)
        if read_range is None:
            self._check(self.L.cmx_ingest_fastq(*args, C.byref(g)), "cmx_ingest_fastq")
        else:
            self._check(self.L.cmx_ingest_fastq_range(*args, C.byref(read_range), C.byref(g)), "cmx_ingest_fastq_range")
        return g, (spans[:2 * g.n_reads].reshape(-1, 2) if want_names else None)

    def set_lanes(self, n):
        self._check(self.L.cmx_set_lanes(self.h, int(n)), "cmx_set_lanes")

    def set_max_read_length(self, n):
        """Resize the context for reads of up to n bases (cmx_set_max_read_length)."""
        self._check(self.L.cmx_set_max_read_length(self.h, int(n)), "cmx_set_max_read_length")

    def timing(self):
        t = Timing()
        self._check(self.L.cmx_last_batch_timing(self.h, C.byref(t)), "cmx_last_batch_timing")
        return t.asdict()

    def trace(self, n_pairs):
        out = np.zeros(n_pairs, dtype=PAIR_TRACE)
        self._check(self.L.cmx_last_batch_trace(self.h, out.ctypes.data, n_pairs), "cmx_last_batch_trace")
        return out

    def postprocess(self, recs):
        recs = np.ascontiguousarray(recs.copy())
        n = C.c_uint64()
        self._check(self.L.cmx_postprocess(self.h, recs.ctypes.data, len(recs), C.byref(n)), "cmx_postprocess")
        return recs[:n.value]

    def postprocess_gpu(self, recs, bcs=None):
        """Sort / dedup / filter on the device; same results as postprocess / postprocess_pairs / postprocess_bc."""
        recs = np.ascontiguousarray(recs.copy())
        n = C.c_uint64()
        if bcs is not None:
            bcs = np.ascontiguousarray(bcs.copy(), dtype=np.uint64)
        self._check(self.L.cmx_postprocess_gpu(self.h, recs.ctypes.data, bcs.ctypes.data if bcs is not None else None, len(recs), C.byref(n)),
                    "cmx_postprocess_gpu")
        return recs[:n.value] if bcs is None else (recs[:n.value], bcs[:n.value])

    def postprocess_bc_bulk_gpu(self, recs, bcs):
        """Barcoded records de-duplicated at bulk level on the device, with the uploaded whitelist's abundances (low-memory
        context that removes duplicates).  Returns (records, barcode keys); raises BulkDedupError with the status."""
        recs = np.ascontiguousarray(recs.copy()); bcs = np.ascontiguousarray(np.array(bcs, dtype=np.uint64).copy())
        n = C.c_uint64()
        rc = self.L.cmx_postprocess_bc_bulk_gpu(self.h, recs.ctypes.data, bcs.ctypes.data, len(recs), C.byref(n))
        if rc != 0:
            raise BulkDedupError("cmx_postprocess_bc_bulk_gpu failed (%d): %s" % (rc, self.L.cmx_last_error(self.h).decode()), rc)
        return recs[:n.value], bcs[:n.value]

    def _allocate(self, fn, what, recs, bcs, distance, seed):
        recs = np.ascontiguousarray(recs.copy())
        if bcs is not None:
            bcs = np.ascontiguousarray(bcs.copy(), dtype=np.uint64)
        n = C.c_uint64()
        st = AllocationStats()
        self._check(fn(self.h, recs.ctypes.data, bcs.ctypes.data if bcs is not None else None, len(recs), int(distance), int(seed), C.byref(n), C.byref(st)), what)
        stats = {f: int(getattr(st, f)) for f, _ in AllocationStats._fields_}
        return recs[:n.value], (bcs[:n.value] if bcs is not None else None), stats

    def allocate_multi_mappings_gpu(self, recs, bcs=None, distance=0, seed=11):
        """--allocate-multi-mappings on the device: Tn5 / sort / dedup, allocation of the multi-mappings (mapq < 4) to their
        uni-mapping neighbourhood, sort, MAPQ filter.  Returns (records, barcode keys or None, stats dict)."""
        return self._allocate(self.L.cmx_allocate_multi_mappings_gpu, "cmx_allocate_multi_mappings_gpu", recs, bcs, distance, seed)

    def allocate_multi_mappings(self, recs, bcs=None, distance=0, seed=11):
        """Host twin of allocate_multi_mappings_gpu (std::mt19937 + std::discrete_distribution)."""
        return self._allocate(self.L.cmx_allocate_multi_mappings, "cmx_allocate_multi_mappings", recs, bcs, distance, seed)

    def postprocess_pairs(self, recs):
        recs = np.ascontiguousarray(recs.copy())
        n = C.c_uint64()
        self._check(self.L.cmx_postprocess_pairs(self.h, recs.ctypes.data, len(recs), C.byref(n)), "cmx_postprocess_pairs")
        return recs[:n.value]

    def format_pairs(self, recs, read_names, lengths, first_read_id=0, names=None):
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        rn = (C.c_char_p * len(read_names))(*[s if isinstance(s, bytes) else s.encode() for s in read_names])
        lens = np.ascontiguousarray(lengths, dtype=np.uint32)
        recs = np.ascontiguousarray(recs)
        n = self.L.cmx_format_pairs(arr, lens.ctypes.data, len(names), recs.ctypes.data, len(recs), rn, first_read_id, None, 0)
        buf = C.create_string_buffer(n + 1)
        self.L.cmx_format_pairs(arr, lens.ctypes.data, len(names), recs.ctypes.data, len(recs), rn, first_read_id, buf, n)
        return buf.raw[:n]

    def format_pairs_gpu(self, recs, read_names, lengths, first_read_id=0, names=None):
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        rn = (C.c_char_p * len(read_names))(*[s if isinstance(s, bytes) else s.encode() for s in read_names])
        lens = np.ascontiguousarray(lengths, dtype=np.uint32)
        recs = np.ascontiguousarray(recs)
        args = (self.h, arr, lens.ctypes.data, len(names), recs.ctypes.data, len(recs), rn, len(read_names), first_read_id)
        n = self.L.cmx_format_pairs_gpu(*args, None, 0)
        if n < 0:
            raise RuntimeError("cmx_format_pairs_gpu: " + self.L.cmx_last_error(self.h).decode())
        buf = C.create_string_buffer(n + 1)
        assert self.L.cmx_format_pairs_gpu(*args, buf, n) == n
        return buf.raw[:n]

    def postprocess_bc(self, recs, bcs):
        recs = np.ascontiguousarray(recs.copy()); bcs = np.ascontiguousarray(bcs.copy(), dtype=np.uint64)
        n = C.c_uint64()
        self._check(self.L.cmx_postprocess_bc(self.h, recs.ctypes.data, bcs.ctypes.data, len(recs), C.byref(n)), "cmx_postprocess_bc")
        return recs[:n.value], bcs[:n.value]

    def format_bed_bc(self, recs, bcs, bc_len, names=None):
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        recs = np.ascontiguousarray(recs); bcs = np.ascontiguousarray(bcs, dtype=np.uint64)
        n = self.L.cmx_format_bed_bc(arr, recs.ctypes.data, bcs.ctypes.data, len(recs), bc_len, None, 0)
        buf = C.create_string_buffer(n + 1)
        self.L.cmx_format_bed_bc(arr, recs.ctypes.data, bcs.ctypes.data, len(recs), bc_len, buf, n)
        return buf.raw[:n]

    def format_bed_bc_tr(self, recs, bcs, bc_len, translation, names=None):
        return format_bed_bc_tr(names or self.names, recs, bcs, bc_len, translation)

    def format_bed_gpu(self, recs, bcs=None, bc_len=0, names=None):
        """BED text written on the device; byte-identical to format_bed / format_bed_bc."""
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        recs = np.ascontiguousarray(recs)
        bp = None
        if bcs is not None:
            bcs = np.ascontiguousarray(bcs, dtype=np.uint64)
            bp = bcs.ctypes.data
        n = self.L.cmx_format_bed_gpu(self.h, arr, recs.ctypes.data, bp, len(recs), bc_len, None, 0)
        if n == -8:
            raise BarcodeNotTranslated(self.L.cmx_last_error(self.h).decode())
        if n < 0:
            raise RuntimeError("cmx_format_bed_gpu: " + self.L.cmx_last_error(self.h).decode())
        buf = C.create_string_buffer(n + 1)
        m = self.L.cmx_format_bed_gpu(self.h, arr, recs.ctypes.data, bp, len(recs), bc_len, buf, n)
        assert m == n
        return buf.raw[:n]

    def format_sam_gpu(self, records, reads1, reads2=None, bcs=None, bc_len=0, first_read_id=0, ref_lengths=None, names=None):
        """SAM text written on the device from SAM cores (bcs: one barcode key per core, None: bulk), with this context's
        parameters and uploaded translation table; byte-identical to format_sam_bc.  reads*: (names, seqs, quals) lists of
        bytes.  ref_lengths defaults to the uploaded sequences' lengths."""
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        lens = np.ascontiguousarray(ref_lengths if ref_lengths is not None else self.ref_lengths, dtype=np.uint32)
        keep = []
        r1, r2 = _sam_read_set(reads1, keep), _sam_read_set(reads2, keep)
        recs = np.ascontiguousarray(records)
        bp = np.ascontiguousarray(bcs, dtype=np.uint64) if bcs is not None else None
        args = (self.h, arr, lens.ctypes.data, len(names), recs.ctypes.data, bp.ctypes.data if bp is not None else None, bc_len, len(recs), C.byref(r1),
                C.byref(r2) if r2 is not None else None, first_read_id)
        n = self.L.cmx_format_sam_gpu(*args, None, 0)
        if n == ERR_BARCODE_TRANSLATE:
            raise BarcodeNotTranslated(self.L.cmx_last_error(self.h).decode())
        if n < 0:
            raise CmxError("cmx_format_sam_gpu failed (%d): %s" % (n, self.L.cmx_last_error(self.h).decode()))
        buf = C.create_string_buffer(n + 1)
        assert self.L.cmx_format_sam_gpu(*args, buf, n) == n
        return buf.raw[:n]

    def format_tagalign(self, recs, names=None):
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        recs = np.ascontiguousarray(recs)
        n = self.L.cmx_format_tagalign(arr, recs.ctypes.data, len(recs), None, 0)
        buf = C.create_string_buffer(n + 1)
        self.L.cmx_format_tagalign(arr, recs.ctypes.data, len(recs), buf, n)
        return buf.raw[:n]

    def format_bed(self, recs, names=None):
        names = names or self.names
        arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
        recs = np.ascontiguousarray(recs)
        n = self.L.cmx_format_bed(arr, recs.ctypes.data, len(recs), None, 0)
        buf = C.create_string_buffer(n + 1)
        self.L.cmx_format_bed(arr, recs.ctypes.data, len(recs), buf, n)
        return buf.raw[:n]

    # ---- stage entry points
    def stage_minimizers(self, seq1, off1, seq2, off2, stride):
        n = len(off1) - 1
        seq1 = np.ascontiguousarray(seq1, dtype=np.uint8); seq2 = np.ascontiguousarray(seq2, dtype=np.uint8)
        off1 = np.ascontiguousarray(off1, dtype=np.uint32); off2 = np.ascontiguousarray(off2, dtype=np.uint32)
        b = Batch(n, _ptr(seq1), _ptr(off1), _ptr(seq2), _ptr(off2), 0, 0)
        h = np.zeros((2 * n, stride), dtype=np.uint64); p = np.zeros((2 * n, stride), dtype=np.uint32)
        cnt = np.zeros(2 * n, dtype=np.int32)
        self._check(self.L.cmx_stage_minimizers(self.h, C.byref(b), h.ctypes.data, p.ctypes.data, cnt.ctypes.data, stride), "cmx_stage_minimizers")
        return h, p, cnt

    def stage_probe(self, hashes):
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        n = len(hashes)
        f = np.zeros(n, dtype=np.uint8); k = np.zeros(n, dtype=np.uint64); v = np.zeros(n, dtype=np.uint64)
        self._check(self.L.cmx_stage_probe(self.h, hashes.ctypes.data, n, f.ctypes.data, k.ctypes.data, v.ctypes.data), "cmx_stage_probe")
        return f, k, v

    def stage_cta_sort(self, keys, tags=None, sm_cap=4096):
        keys = np.ascontiguousarray(keys, dtype=np.uint64).copy()
        tags = None if tags is None else np.ascontiguousarray(tags, dtype=np.uint8).copy()
        self._check(self.L.cmx_stage_cta_sort(self.h, keys.ctypes.data, None if tags is None else tags.ctypes.data, len(keys), sm_cap), "cmx_stage_cta_sort")
        return keys, tags

    def stage_correct_barcodes(self, barcodes, quals, bc_len):
        """CorrectBarcodeAt for n barcodes (uint8 arrays of n * bc_len ASCII bytes) against the uploaded whitelist, with the
        kernels map_batch runs.  Returns (keys uint64[n], ok uint8[n], n_in_whitelist, n_corrected)."""
        barcodes = np.ascontiguousarray(barcodes, dtype=np.uint8); quals = np.ascontiguousarray(quals, dtype=np.uint8)
        n = barcodes.size // bc_len
        keys = np.zeros(n, dtype=np.uint64); ok = np.zeros(n, dtype=np.uint8)
        n_in, n_cor = C.c_uint64(), C.c_uint64()
        self._check(self.L.cmx_stage_correct_barcodes(self.h, barcodes.ctypes.data, quals.ctypes.data, n, bc_len, keys.ctypes.data, ok.ctypes.data,
                                                      C.byref(n_in), C.byref(n_cor)), "cmx_stage_correct_barcodes")
        return keys, ok, n_in.value, n_cor.value

    def stage_banded_align(self, e, read_len, patterns, texts):
        patterns = np.ascontiguousarray(patterns, dtype=np.uint8); texts = np.ascontiguousarray(texts, dtype=np.uint8)
        n = texts.size // read_len
        err = np.zeros(n, dtype=np.int32); endp = np.zeros(n, dtype=np.int32)
        self._check(self.L.cmx_stage_banded_align(self.h, e, read_len, patterns.ctypes.data, texts.ctypes.data, n, err.ctypes.data, endp.ctypes.data), "cmx_stage_banded_align")
        return err, endp
