/* chromap_b200 — C ABI of the H100-native (sm_90a) replacement for Chromap's per-read mapping hot path.
 *
 * The reference (haowenz/chromap) has NO plugin / FFI interface: it is one executable whose hot path is
 * the body of the OpenMP taskloop in src/chromap.h:892-1143 (paired-end).  This header DEFINES the
 * boundary a maintainer would bind (INTEGRATION.md shows the call sites to replace).  Every entry point
 * cites the reference interface it replaces (paths relative to the reference's src/).
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success or a negative
 * cmx_status; nothing exits or throws across the ABI (the reference calls exit(-1), utils.h:71-74).
 * There is no CPU fallback: without a CUDA device cmx_create() fails with CMX_ERR_NO_DEVICE.
 */
#ifndef CHROMAP_B200_H_
#define CHROMAP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  CMX_OK = 0,
  CMX_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product path refuses to run */
  CMX_ERR_CUDA = -2,        /* a CUDA runtime call failed; see cmx_last_error() */
  CMX_ERR_INVALID = -3,     /* bad argument / unsupported parameter combination */
  CMX_ERR_STATE = -4,       /* index or reference not uploaded yet */
  CMX_ERR_OVERFLOW = -5,    /* a pair exceeded even the large scratch tier (reported, never silent) */
  CMX_ERR_IO = -6,
  CMX_ERR_READ_RANGE = -7,  /* --read-format ranges the reference cuts in an undefined way (see cmx_read_range) */
  CMX_ERR_BARCODE_TRANSLATE = -8 /* a barcode segment has no entry in the --barcode-translate table */
} cmx_status;

/* POD mirror of the MappingParameters fields the path reads (mapping_parameters.h:18-78). */
typedef struct {
  int32_t error_threshold;        /* -e   (8)   */
  int32_t min_num_seeds;          /* -s   (2)   */
  int32_t max_seed_freq0;         /* -f a (500) */
  int32_t max_seed_freq1;         /* -f b (1000)*/
  int32_t max_num_best_mappings;  /* -n   (1)   */
  int32_t max_insert_size;        /* -l   (1000)*/
  int32_t mapq_threshold;         /* -q   (30)  */
  int32_t min_read_length;        /* --min-read-length (30) */
  int32_t drop_repetitive_reads;  /* (500000) */
  int32_t trim_adapters;
  int32_t remove_pcr_duplicates;
  int32_t tn5_shift;
  int32_t split_alignment;        /* --split-alignment (Hi-C); requires output_format == 5 */
  int32_t low_memory_mode;
  int32_t output_format;          /* 1 = BED, 2 = TagAlign (same records), 4 = SAM cores (cmx_sam_record), 5 = pairs (mapping_parameters.h:9-16) */
  int32_t batch_size;             /* pairs per reference batch (chromap.h:182: 500000); fixes the
                                     taskloop chunking that seeds multi-mapper sampling */
  int32_t max_read_length;        /* upper bound on read length in any batch (sizing), default 160 */
  int32_t single_end;             /* 1 = single-end reads (chromap -1 only; MapSingleEndReads, chromap.h:218-634): cmx_batch.seq2/off2
                                     are NULL, records are MappingWithoutBarcode (both alignment lengths 0). BED, non-split only */
} cmx_params;

void cmx_default_params(cmx_params *p);
/* chromap_driver.cc:247-275.  preset = "chip" | "atac" | "hic" | "".  -3 if unknown. */
int cmx_apply_preset(cmx_params *p, const char *preset);

typedef struct cmx_ctx cmx_ctx; /* one per GPU */

/* Replaces the Chromap(MappingParameters) constructor + stage objects (chromap.h:176-215,803-812). */
int cmx_create(cmx_ctx **out, int device, const cmx_params *params);
void cmx_destroy(cmx_ctx *ctx);
const char *cmx_last_error(const cmx_ctx *ctx);

/* Replaces SequenceBatch::LoadAllSequences for the reference (chromap.h:641-644, sequence_batch.cc:84):
 * n_seq sequences, bases as loaded (ASCII, case preserved), concatenated; offsets[n_seq+1]. Host buffers
 * are borrowed for the duration of the call. */
int cmx_upload_reference(cmx_ctx *ctx, uint32_t n_seq, const uint64_t *offsets, const char *concat_ascii);

/* Replaces Index::Load (index.cc:132-169): the khash arrays of the index file (khash.h:358-373) and the
 * occurrence table, re-laid-out on the device (layout is free; every lookup answers identically). */
int cmx_upload_index(cmx_ctx *ctx, int k, int w, uint32_t n_buckets, const uint32_t *flags,
                     const uint64_t *keys, const uint64_t *vals, const uint64_t *occ, uint32_t n_occ);
/* Replaces Index::Construct (index.cc:12-89) on the device, from the uploaded reference. */
int cmx_build_index(cmx_ctx *ctx, int k, int w);
/* Download the index in the reference's file layout pieces (for Index::Save, index.cc:91-130).
 * Pass NULL buffers to query sizes. */
int cmx_download_index(cmx_ctx *ctx, uint32_t *n_buckets, uint32_t *n_keys, uint32_t *flags,
                       uint64_t *keys, uint64_t *vals, uint32_t *n_occ, uint64_t *occ);
int cmx_index_info(const cmx_ctx *ctx, int *k, int *w, uint64_t *n_keys, uint64_t *n_occ,
                   uint64_t *table_slots);

/* scATAC barcode whitelist with the abundances of ComputeBarcodeAbundance (chromap.cc:388-548, a host pre-pass over the
 * barcode file): n distinct 2-bit packed keys (GenerateSeedFromSequence, utils.h:107-126), their counts among the
 * sampled barcodes and the sample size.  Enables CorrectBarcodeAt (chromap.cc:572-799) inside cmx_map_batch_pe.
 * err_threshold = --bc-error-threshold: 0, 1 or 2 substitutions (at 2 a barcode may carry up to two Ns); any other value
 * returns CMX_ERR_INVALID, since the reference would leave the Ns beyond the second in the key as A.
 * prob_threshold = --bc-probability-threshold. */
int cmx_upload_barcode_whitelist(cmx_ctx *ctx, const uint64_t *keys, const uint32_t *counts, uint64_t n, uint64_t num_sample,
                                 uint32_t bc_len, int err_threshold, double prob_threshold, int output_not_in_whitelist);

/* One batch of read pairs = the inputs of the taskloop (read_batch1, read_batch2; chromap.h:892).
 * Bases are ASCII exactly as in the FASTQ; pair i's mates are seq1[off1[i]..off1[i+1]) and
 * seq2[off2[i]..off2[i+1]).  on_device != 0: all four pointers are device pointers. */
typedef struct {
  uint32_t n_pairs;
  const char *seq1;
  const uint32_t *off1; /* n_pairs + 1 */
  const char *seq2;
  const uint32_t *off2;   /* n_pairs + 1 */
  uint32_t first_read_id; /* running read counter (sequence_batch.cc:38-39) */
  int32_t on_device;
  /* scATAC (optional, NULL for bulk data): one cell barcode + its qualities per pair, bc_len bytes each
   * (barcode_batch of chromap.h:892-909); host or device pointers like the reads. */
  const char *bc_seq;
  const char *bc_qual;
  uint32_t bc_len;
} cmx_batch;

/* PairedEndMappingWithoutBarcode (bed_mapping.h:170-238) without the vptr, plus rid. 24 bytes. */
typedef struct {
  uint32_t read_id;
  uint32_t rid;
  uint32_t fragment_start;
  uint16_t fragment_length;
  uint8_t mapq;
  uint8_t direction; /* 1 = read 1 on + strand */
  uint8_t is_unique;
  uint8_t num_dups;
  uint16_t positive_alignment_length;
  uint16_t negative_alignment_length;
} cmx_pe_record;

/* PairsMapping (pairs_mapping.h:11-49) without the read name: what --preset hic emits (mapping_generator.cc:169-210).
 * 24 bytes; written into the same record buffer when output_format == 5 (pairs). */
typedef struct {
  uint32_t read_id;
  uint32_t rid1, rid2;
  uint32_t pos1, pos2;      /* 0-based 5' positions, (rid1, pos1) <= (rid2, pos2) */
  uint8_t strand1, strand2; /* 1 = + */
  uint8_t mapq, is_unique;
} cmx_pairs_record;

/* output_format == 4 (MAPPINGFORMAT_SAM): what the SAM writer needs from the device for one reported pair (paired-end) or
 * read (single-end, index 0 only): the spans and CIGARs ksw_semi_global3 gives (ksw.cc:505-626 through
 * mapping_generator.h:723-760,807-855), MAPQ computed from those spans, strands.  Flags, TLEN, NM / MD and the text follow on
 * the host from these fields (mapping_generator.h:613-640, mapping_generator.cc:84-107, alignment.cc:85-139).  Written into
 * the records buffer, which must then hold capacity * sizeof(cmx_sam_record) bytes.  Non-split, reads <= 160 bases. */
#define CMX_SAM_MAX_CIGAR 24
typedef struct {
  uint32_t read_id, rid;
  uint32_t pos[2], end[2]; /* 0-based inclusive reference span of mate 1 / mate 2 */
  uint8_t strand[2];       /* 1 = + */
  uint8_t mapq, is_unique;
  uint8_t secondary;       /* not the first reported mapping of this read (BAM_FSECONDARY) */
  uint8_t n_cigar[2];
  uint8_t overflow;        /* the call also returns CMX_ERR_OVERFLOW: read or CIGAR beyond the fixed record */
  uint32_t cigar[2][CMX_SAM_MAX_CIGAR]; /* BAM encoding: length << 4 | op, M = 0, I = 1, D = 2 */
} cmx_sam_record;

typedef struct {
  cmx_pe_record *records; /* caller-owned, capacity >= n_pairs * max_num_best_mappings (cmx_pairs_record when pairs) */
  uint64_t capacity;
  uint64_t n_records;    /* out */
  int32_t on_device;     /* records is a device pointer (n_records still returned on the host) */
  /* out: counters the reference prints (chromap.cc:808-823) */
  uint64_t n_mapped_pairs, n_uniquely_mapped_pairs, n_candidates, n_overflow_pairs;
  /* scATAC: barcode key (2 bits per base, after correction) of every returned record, same capacity as `records`
   * (host pointer; may be NULL), and the counters of chromap.cc:801-805 */
  uint64_t *barcode_keys;
  uint64_t n_barcodes_in_whitelist, n_barcodes_corrected;
} cmx_records;

/* Replaces the taskloop body over one batch, chromap.h:892-1143: trimming, minimizers, index probe,
 * candidate clustering, mate supplementation, paired-end filter, banded verification, pairing,
 * multi-mapper sampling, start-coordinate traceback, MAPQ, record emit.  Records come back in read
 * order.  Synchronous: returns when the records are in `out`. `stream` (cudaStream_t) may be NULL. */
int cmx_map_batch_pe(cmx_ctx *ctx, const cmx_batch *in, cmx_records *out, void *stream);

/* Post-processing on the device (mapping_processor.h:100-202, mapping_writer.h:166-376,
 * chromap.h:1305-1355): sort by (rid, record order), duplicate removal, Tn5 shift, MAPQ filter.
 * In place on host records; returns the surviving count in *n_out. */
int cmx_postprocess(cmx_ctx *ctx, cmx_pe_record *records, uint64_t n, uint64_t *n_out);
/* Pairs post-processing (low-memory merge, mapping_writer.h:166-376 with PairsMapping order pairs_mapping.h:40-49) and
 * text with header (mapping_writer.cc:381-421).  read_names[i] = name of read 1 of pair (read_id - first_read_id). */
int cmx_postprocess_pairs(cmx_ctx *ctx, cmx_pairs_record *records, uint64_t n, uint64_t *n_out);
int64_t cmx_format_pairs(const char *const *names, const uint32_t *lengths, uint32_t n_seq, const cmx_pairs_record *records, uint64_t n,
                         const char *const *read_names, uint32_t first_read_id, char *buf, int64_t cap);
/* scATAC post-processing and BED text: records ordered / de-duplicated with the barcode in the key
 * (PairedEndMappingWithBarcode, bed_mapping.h:116-167; cell-level dedup as the atac preset sets it) and written as
 * `chrom start end barcode num_dups` (mapping_writer.cc:127-137). */
int cmx_postprocess_bc(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n, uint64_t *n_out);
/* Multi-GPU (SURVEY.md 8e): one process per GPU, every process owns whole reference batches and calls this library on its own
 * device; nothing in the hot path crosses GPUs.  The one exchange step -- duplicate removal over the whole run -- is a single
 * NCCL all-gather of 16-byte tuples followed by the local decision above; it is driven from chromap_b200/distributed.py over
 * torch.distributed (which owns the communicator), so there is deliberately no C entry point for it. */

/* The same three routines on the device (LSD radix sort over the reference's record order + run resolution), in place on
 * host buffers: `records` is cmx_pairs_record[] when the context emits pairs, cmx_pe_record[] otherwise; barcode_keys
 * is NULL for bulk data.  Replaces the sort / merge of mapping_processor.h:100-202 and mapping_writer.h:166-376 the
 * same way; results are identical to the host routines.  n < 2^31 per call. */
int cmx_postprocess_gpu(cmx_ctx *ctx, void *records, uint64_t *barcode_keys, uint64_t n, uint64_t *n_out);

/* --allocate-multi-mappings: counts of one call (the reference's log lines, mapping_processor.h:363,431-435,502-504). */
typedef struct {
  uint64_t n_multi;            /* multi-mappings (mapq < 4) after duplicate removal: "Got all X multi-mappings!" */
  uint64_t n_allocated;        /* reads given one of their candidates */
  uint64_t n_without_overlap;  /* reads whose weight sum is 0 (dropped) */
  uint64_t n_draws;            /* reads that consumed two generator outputs (>= 2 candidates, non-zero sum) */
  uint64_t n_uni_after, n_multi_after;  /* is_unique split of the allocated set, before the MAPQ filter */
} cmx_allocation_stats;
/* In-memory post-processing with multi-mapping allocation (chromap.h:1322-1355 with allocate_multi_mappings): Tn5 shift, sort,
 * duplicate removal (keeping the last of a run), AllocateMultiMappings (mapping_processor.h:319-440: each read with mapq < 4
 * keeps one candidate drawn with weights = the uni-mappings within `distance` of it, from one std::mt19937(seed); reads
 * without any such uni-mapping are dropped), sort, MAPQ filter.  Bulk or barcoded (barcode_keys != NULL), paired-end or
 * single-end records, in place on host buffers like cmx_postprocess_gpu; *n_out = the records left.  CMX_ERR_INVALID, with
 * the reason in cmx_last_error() and the records untouched, for a low-memory context (the reference never allocates there),
 * a pairs or SAM context, distance < 0, n >= 2^31, or a record set without any multi-mapping (the reference aborts). */
int cmx_allocate_multi_mappings_gpu(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n,
                                    int32_t distance, int32_t seed, uint64_t *n_out, cmx_allocation_stats *stats);
/* Host twin (std::mt19937 + std::discrete_distribution): the same results, refusals and counts. */
int cmx_allocate_multi_mappings(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n,
                                int32_t distance, int32_t seed, uint64_t *n_out, cmx_allocation_stats *stats);
int64_t cmx_format_bed_bc(const char *const *names, const cmx_pe_record *records, const uint64_t *barcode_keys, uint64_t n, uint32_t bc_len,
                          char *buf, int64_t cap);
/* BED text (mapping_writer.cc:75-83); names = n_seq C strings.  Returns bytes (or needed size if buf NULL). */
int64_t cmx_format_bed(const char *const *names, const cmx_pe_record *records, uint64_t n, char *buf,
                       int64_t cap);
/* The same text written on the device (also the barcoded form when barcode_keys != NULL): per-line lengths, exclusive
 * scan, one thread per line; host buffers in and out, byte-identical to cmx_format_bed / cmx_format_bed_bc.
 * buf == NULL returns the length only; < 0 on error. */
/* --TagAlign (MAPPINGFORMAT_TAGALIGN = 2, mapping_writer.cc:84-110) for paired-end records: the same records as BED, one line
 * per mate.  Single-end TagAlign is the BED text. */
int64_t cmx_format_tagalign(const char *const *names, const cmx_pe_record *records, uint64_t n, char *buf, int64_t cap);
int64_t cmx_format_bed_gpu(cmx_ctx *ctx, const char *const *names, const cmx_pe_record *records, const uint64_t *barcode_keys,
                           uint64_t n, uint32_t bc_len, char *buf, int64_t cap);

/* --barcode-translate (BarcodeTranslator, barcode_translator.h; loaded by the writer's constructor, mapping_writer.h:39-42):
 * the barcode field of barcoded BED lines becomes the TO strings of the key's segments.  A table file has lines TO<sep>FROM,
 * <sep> the first ',' or '\t'; the key of FROM is GenerateSeedFromSequence (utils.h:111-129).  With L the FROM length, a
 * barcode of bc_len bases has nseg = bc_len / L segments, segment s being the L bases that end (nseg - 1 - s) * L bases
 * before its last (the leading bc_len mod L bases are ignored); the field is their TO strings joined by '-', empty when
 * nseg == 0.  Order and duplicate removal keep using the untranslated key. */
typedef struct {
  uint64_t n;        /* distinct FROM keys */
  uint64_t *keys;    /* [n], in the order of their first line */
  uint64_t *to_off;  /* [n + 1]: TO of keys[i] = to[to_off[i] .. to_off[i + 1]), from the key's last line */
  char *to;          /* TO strings, concatenated (not NUL-terminated) */
  uint32_t from_len; /* L, 1..31 */
} cmx_barcode_translation;
/* Host only.  text = the file's bytes (inflated), one table per file.  Refuses with CMX_ERR_INVALID, the reason and the
 * 1-based line in err (err_cap bytes, may be NULL), what the reference reads in an undefined or accidental way: no line at
 * all; an empty line, a line without a separator or with an empty FROM; a FROM byte outside ACGTacgt (N, the '\r' of CRLF);
 * FROMs of different lengths; L >= 32; a line longer than 510 bytes before its newline (gzgets' 512-byte buffer splits it);
 * a NUL byte.  A repeated FROM takes the TO of its last line; TO may be empty; the last line needs no newline.
 * On success *out owns its arrays: release them with cmx_free_barcode_translation. */
int cmx_parse_barcode_translation(const char *text, uint64_t n_bytes, cmx_barcode_translation *out, char *err, uint64_t err_cap);
void cmx_free_barcode_translation(cmx_barcode_translation *t);
/* The table on the device (HBM), replacing the previous one; NULL removes it.  While one is uploaded, cmx_format_bed_gpu with
 * barcode_keys writes translated fields, and returns CMX_ERR_BARCODE_TRANSLATE before writing any text when a segment has no
 * entry (where the reference prints "Barcode does not exist in the translation table." and exits 255, after part of the
 * file); cmx_last_error() then gives the number of such segments and the first barcode, in output order, that has one. */
int cmx_upload_barcode_translation(cmx_ctx *ctx, const cmx_barcode_translation *translation);
/* Host twin of the translated text: cmx_format_bed_bc with `translation` applied (NULL: exactly cmx_format_bed_bc).  Returns
 * the bytes (or the needed size if buf is NULL), CMX_ERR_BARCODE_TRANSLATE with nothing written if a segment has no entry. */
int64_t cmx_format_bed_bc_tr(const char *const *names, const cmx_pe_record *records, const uint64_t *barcode_keys, uint64_t n, uint32_t bc_len,
                             const cmx_barcode_translation *translation, char *buf, int64_t cap);
/* Pairs text (header + lines of cmx_format_pairs) with the lines written on the device.  read_names[i] is the name of read
 * first_read_id + i (n_read_names of them). */
int64_t cmx_format_pairs_gpu(cmx_ctx *ctx, const char *const *names, const uint32_t *lengths, uint32_t n_seq, const cmx_pairs_record *records,
                             uint64_t n, const char *const *read_names, uint64_t n_read_names, uint32_t first_read_id, char *buf, int64_t cap);

/* ---- stage-level entry points: fixture-level parity tests and ncu isolation ------------------- */
/* MinimizerGenerator::GenerateMinimizers (minimizer_generator.cc:7-139) for every read of a host batch.
 * out_hash/out_pos hold n_reads*stride entries (stride = max_read_length); out_n the per-read count.
 * out_pos = (end_position << 1) | strand.  Reads are numbered 2*pair + mate. */
int cmx_stage_minimizers(cmx_ctx *ctx, const cmx_batch *in, uint64_t *out_hash, uint32_t *out_pos,
                         int32_t *out_n, uint32_t stride);
/* kh_get (khash.h:232-245) for n minimizer hashes: found[i], key[i] (hash<<1|singleton), val[i]. */
int cmx_stage_probe(cmx_ctx *ctx, const uint64_t *hashes, uint64_t n, uint8_t *found, uint64_t *key,
                    uint64_t *val);
/* BandedAlignPatternToText (alignment.cc:141-192) on n (pattern, text) problems of equal read_len:
 * patterns n*(read_len+2e) bytes, texts n*read_len bytes. */
int cmx_stage_banded_align(cmx_ctx *ctx, int e, int read_len, const char *patterns, const char *texts,
                           uint64_t n, int32_t *num_errors, int32_t *end_pos);
/* The overflow tiers' CTA-cooperative bitonic sort on n keys (tags != NULL: (count desc, position asc) candidate
 * order, mapping_metadata.h:65-68 / candidate.h:23-33); sm_cap = shared-memory tile (power of two <= 4096). */
int cmx_stage_cta_sort(cmx_ctx *ctx, uint64_t *keys, uint8_t *tags, uint32_t n, uint32_t sm_cap);
/* CorrectBarcodeAt (chromap.cc:572-799) for n host barcodes of bc_len bases (ASCII bases and qualities, n*bc_len bytes each)
 * against the uploaded whitelist, with the kernels cmx_map_batch_pe runs: out_key[i] = the 2-bit key afterwards, out_ok[i] =
 * 1 if it is in the whitelist or corrected (or --output-mappings-not-in-whitelist), and the two counters of the batch. */
int cmx_stage_correct_barcodes(cmx_ctx *ctx, const char *bc_seq, const char *bc_qual, uint64_t n, uint32_t bc_len,
                               uint64_t *out_key, uint8_t *out_ok, uint64_t *n_in_whitelist, uint64_t *n_corrected);
/* Per-pair counters after a full cmx_map_batch_pe (same fields as the oracle's trace). */
typedef struct {
  int32_t n_minimizers[2];
  int32_t n_pos_candidates_gen[2], n_neg_candidates_gen[2];
  int32_t n_pos_candidates[2], n_neg_candidates[2];
  int32_t n_pos_mappings[2], n_neg_mappings[2];
  int32_t min_errors[2], second_min_errors[2], n_best[2], n_second_best[2];
  uint32_t repetitive_seed_length[2];
  int32_t supplement_result;
  int32_t min_sum_errors, second_min_sum_errors, n_best_pairs, n_second_best_pairs;
  int32_t n_records;
  int32_t trimmed_len[2];
} cmx_pair_trace;
int cmx_last_batch_trace(cmx_ctx *ctx, cmx_pair_trace *out, uint32_t n_pairs);

/* Kernel timing of the last cmx_map_batch_pe (CUDA events on the launching stream), in ms. */
typedef struct {
  float h2d_ms, seed_ms, pair_candidates_ms, verify_ms, pairing_ms, select_ms, emit_ms, d2h_ms, total_ms;
  float front_ms, reserved_ms, cluster_ms;  /* tier-0 parts of seed_ms: front_ms = the fused front-end kernel (length filter +
                                             * minimizers + index probe, seed_front.cuh), cluster_ms = hit lists + clustering;
                                             * seed_ms - front_ms - cluster_ms = seeding of the overflow tiers */
  uint64_t n_minimizers, n_probe_steps, n_found, n_occ_reads, n_verified, n_launches;
  uint64_t tier_pairs[3];      /* pairs processed per scratch tier */
  uint64_t escalations[8];     /* tier-0 escalations by cause (see Counters::ovf_reason) */
} cmx_timing;
int cmx_last_batch_timing(cmx_ctx *ctx, cmx_timing *out);

/* FASTQ text -> packed reads on the device (the loader's side of the path: SequenceBatch::LoadBatch + kseq_read,
 * sequence_batch.cc:9-60, kseq.h:177-222, for 4-line FASTQ).  `text` (host) must hold whole records: cmx_fastq_cut returns
 * how many bytes the first min(max_records, complete) records take.  The result lives in the context's ingest buffers of
 * `slot` (0..5, independent sets so that three files can be double-buffered) until the next call on that slot, in the layout
 * cmx_batch takes with on_device = 1.  name_spans (optional, host, 2 x n_reads u32): start and length of each read name
 * in `text`.  Anything that is not plain 4-line FASTQ (multi-line records, FASTA, empty reads) returns CMX_ERR_INVALID:
 * the caller falls back to its own reader. */
typedef struct {
  uint32_t n_reads;
  const char *seq;      /* device: bases of all reads, concatenated */
  const uint32_t *off;  /* device: n_reads + 1 offsets into seq */
  const char *qual;     /* device: qualities in the same layout (NULL unless want_qual) */
  uint32_t min_len, max_len;
} cmx_ingested;
uint64_t cmx_fastq_cut(const char *text, uint64_t n_bytes, uint32_t max_records, uint32_t *n_records);
int cmx_ingest_fastq(cmx_ctx *ctx, int slot, const char *text, uint64_t n_bytes, int want_qual, uint32_t *name_spans, cmx_ingested *out);

/* --read-format (chromap.cc:825-865, sequence_effective_range.h:20-118): the part of every read of one file that is kept.
 * Ranges are 0-based and inclusive, concatenated in order; end == -1 is the read's last base.  reverse = 1 ('-' strand):
 * after the cut the bases are complemented (ACGTacgt -> upper-case complement, any other byte -> N, utils.h:87-100) and
 * reversed, the qualities reversed.  {1, {0}, {-1}, 0} keeps the whole read.
 * Only cuts whose result the reference defines are representable: 1..CMX_MAX_READ_RANGES ranges, 0 <= start <= end,
 * ascending and disjoint, -1 in the last range only (Replace copies in place: a range that reaches back would read bytes
 * already overwritten). */
#define CMX_MAX_READ_RANGES 8
typedef struct {
  uint32_t n;
  int32_t start[CMX_MAX_READ_RANGES], end[CMX_MAX_READ_RANGES];
  int32_t reverse;
} cmx_read_range;
/* Host only.  Parses "r1|r2|bc:start:end[:+|-]" fields separated by commas (start >= 0 and end >= start, or end == -1);
 * fields of one file append ranges, the last strand given wins, a file named in no field keeps its whole read ("" = no
 * cut at all).  CMX_ERR_INVALID for anything outside that grammar (the reference's hand parser accepts some such strings,
 * with meanings that are artifacts of its loop); CMX_ERR_READ_RANGE for ranges of one file that are not representable
 * above (the reference runs them, with an output that depends on its in-place copy). */
int cmx_parse_read_format(const char *fmt, cmx_read_range *r1, cmx_read_range *r2, cmx_read_range *bc);
/* Host only: the cut of one read in place (SequenceEffectiveRange::Replace); qual (may be NULL) gets the same ranges and
 * order, not complemented.  Returns the new length; 0 if nothing is left (start >= len in the last, open-ended range);
 * CMX_ERR_READ_RANGE if an explicit end is at or past len (the reference then reads past the string); CMX_ERR_INVALID for
 * a range that is not representable. */
int64_t cmx_apply_read_range(const cmx_read_range *range, char *seq, char *qual, uint32_t len);
/* cmx_ingest_fastq with every record cut by `range` on the device (NULL or the whole read: exactly cmx_ingest_fastq).
 * min_len / max_len are the cut lengths.  CMX_ERR_READ_RANGE, with the counts in cmx_last_error(), if a record is too short
 * for an explicit end or empty after the cut. */
int cmx_ingest_fastq_range(cmx_ctx *ctx, int slot, const char *text, uint64_t n_bytes, int want_qual, uint32_t *name_spans, const cmx_read_range *range,
                           cmx_ingested *out);

/* SAM text from the cores (host only, no device): expands them to one line per mate, puts them in SAMMapping's order,
 * removes duplicates / filters by MAPQ as the context's parameters say (sam_mapping.h:188-199, mapping_processor.h:161-202,
 * mapping_writer.h:166-376,405-437) and writes the @SQ header + lines of mapping_writer.cc:312-356 (flags, mate fields, TLEN,
 * SEQ / QUAL of the mapped strand, NM / MD from the CIGAR).  reads1 / reads2: names, bases and qualities (qual may be NULL)
 * of reads first_read_id .. ; reads2 == NULL for single-end.  buf == NULL returns the length; < 0 on error. */
typedef struct {
  const char *const *names; /* [n_reads] */
  const char *seq;          /* bases, concatenated */
  const uint64_t *off;      /* [n_reads + 1] */
  const char *qual;         /* qualities in the same layout, or NULL */
} cmx_read_set;
int64_t cmx_format_sam(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const char *ref_concat,
                       const uint64_t *ref_offsets, const cmx_sam_record *records, uint64_t n, const cmx_read_set *reads1,
                       const cmx_read_set *reads2, uint32_t first_read_id, char *buf, int64_t cap);
/* The same for barcoded runs (host only): barcode_keys[i] (NULL: exactly cmx_format_sam) is the cell barcode key of core i, as
 * cmx_map_batch_pe returns it; it joins the order (rid, pos, barcode, mrid, mpos, read 1, mapq, read id) and the duplicate
 * test (pos, rid, barcode, read 1, mrid, mpos) of sam_mapping.h:188-199, and every line ends in "\tCB:Z:<field>"
 * (mapping_writer.cc:350-354), the field being what cmx_format_bed_bc_tr writes for the key (translation NULL: its bc_len
 * bases).  Returns -2 for an overflowed core, -3 for a CIGAR longer than its read, CMX_ERR_BARCODE_TRANSLATE with nothing
 * written for a barcode segment without an entry in `translation`, -1 for bad arguments. */
int64_t cmx_format_sam_bc(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const char *ref_concat,
                          const uint64_t *ref_offsets, const cmx_sam_record *records, const uint64_t *barcode_keys, uint32_t bc_len, uint64_t n,
                          const cmx_read_set *reads1, const cmx_read_set *reads2, uint32_t first_read_id,
                          const cmx_barcode_translation *translation, char *buf, int64_t cap);
/* The SAM text written on the device, byte-identical to cmx_format_sam_bc (barcode_keys NULL: cmx_format_sam) with the
 * context's parameters (duplicate rule, MAPQ threshold) and, for barcoded cores, the translation table of
 * cmx_upload_barcode_translation.  NM / MD are computed against the uploaded reference.  Host buffers in and out; the @SQ
 * header is written by the host.  Cores, keys, reads and the sort's scratch are resident on the device for the call (232 B per
 * core + 26 B per line + the reads' bases, qualities and names + 16 B per read; see DESIGN.md): a call that does not fit returns
 * -1, as does any other device failure.  -2, -3 and CMX_ERR_BARCODE_TRANSLATE as the host twin.  buf == NULL returns the length. */
int64_t cmx_format_sam_gpu(cmx_ctx *ctx, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const cmx_sam_record *records,
                           const uint64_t *barcode_keys, uint32_t bc_len, uint64_t n, const cmx_read_set *reads1, const cmx_read_set *reads2,
                           uint32_t first_read_id, char *buf, int64_t cap);

/* --PAF (MAPPINGFORMAT_PAF = 3) text from the BED-path records (host only): PAFMapping / PairedPAFMapping hold the same
 * fields plus read names and the (trimmed) read lengths; order, duplicate rule, Tn5 shift and MAPQ filter are those types'
 * own (paf_mapping.h), reproduced with the quirks of mapping_generator.cc:146-167.  Takes the records as cmx_map_batch_pe
 * returned them (not post-processed).  names2 == NULL: single-end.  buf == NULL returns the length; < 0 on error. */
int64_t cmx_format_paf(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, const cmx_pe_record *records, uint64_t n,
                       const char *const *names1, const uint16_t *lengths1, const char *const *names2, const uint16_t *lengths2,
                       uint32_t first_read_id, char *buf, int64_t cap);


/* Page-lock (pin) a host buffer the caller owns, so that cmx_ingest_fastq / cmx_map_batch_pe copy from it at PCIe speed and
 * asynchronously (cudaHostRegister / cudaHostUnregister).  Optional: unpinned buffers work, slower.  No counterpart in the
 * reference (its loader hands kseq buffers to the mapping threads directly, sequence_batch.cc:9-60). */
int cmx_host_register(void *ptr, uint64_t bytes);
int cmx_host_unregister(void *ptr);

/* Concurrency of one cmx_map_batch_pe call (no counterpart in the reference, whose knob is -t): a call that carries
 * several whole reference batches is cut into up to n_lanes (1..4, default 4) groups of batches that run the whole
 * pipeline on their own streams, so the latency-bound kernels of one group overlap the issue-bound kernels of
 * another.  Results do not depend on it.  With 1 lane the kernels of a call run back to back on one stream and
 * cmx_timing's stage times are exclusive; with more lanes they are sums over overlapping streams.  Changing the
 * count releases the lanes' scratch tiers (they grow again at the next call), so device memory follows the new split. */
int cmx_set_lanes(cmx_ctx *ctx, int n_lanes);


/* ---- multi-GPU: the one exchange step (SURVEY.md 8e) ---------------------------------------------------------------------
 * One process per GPU; read batches are sharded over the ranks with no data-path collective.  Duplicate removal is defined
 * over the whole run (the reference's low-memory merge, mapping_writer.h:166-376), so after mapping every rank packs its
 * records into 16-byte tuples {rid | start, length | mapq | direction | unique | read_id} (24 bytes with a cell barcode), ONE
 * ncclAllGather moves them over NVLink (preceded by an 8-byte all-gather of the counts that sizes it), and every rank sorts
 * the gathered tuples on its GPU and decides which of ITS OWN records survive: the first record in the reference's order
 * carrying the group's highest MAPQ (mapping_writer.h:268-270), duplicate count saturating at 255 (:282-284), MAPQ filter
 * afterwards (:281).  The reference is single-process: there is no call site this replaces; it takes the place of the
 * duplicate test inside OutputMappingsInVector / the temp-file merge (mapping_writer.h:254-287) for a sharded run.
 * NCCL is loaded with dlopen at the first call (no link-time dependency); CMX_ERR_STATE if it is not there. */
int cmx_comm_unique_id(void *id128);                                             /* rank 0: ncclGetUniqueId, 128 bytes */
int cmx_comm_init(cmx_ctx *ctx, int n_ranks, int rank, const void *id128);       /* ncclCommInitRank on the context's device */
int cmx_comm_destroy(cmx_ctx *ctx);
typedef struct {
  float pack_ms, allgather_ms, resolve_ms;   /* CUDA events on the context's stream */
  uint64_t bytes_sent, bytes_received;       /* tuple bytes this rank contributed / received in the all-gather */
  uint64_t n_global;                         /* records of all ranks */
  uint32_t n_ranks, pad;
} cmx_exchange_stats;
/* records (and barcode_keys, NULL for bulk data): this rank's cmx_pe_record array, host or device (on_device); paired-end,
 * low-memory mode (every preset that removes duplicates).  out_records / out_barcode_keys (same kind of memory, capacity n):
 * this rank's survivors in the reference's order, num_dups set, MAPQ-filtered, Tn5 NOT yet applied. */
int cmx_dedup_exchange(cmx_ctx *ctx, const void *records, const uint64_t *barcode_keys, uint64_t n, int on_device, void *out_records,
                       uint64_t *out_barcode_keys, uint64_t *n_out, cmx_exchange_stats *stats);
/* The same step as a range shuffle (a sample sort): the records' key word rid << 32 | fragment_start is range-partitioned over
 * the ranks (splitters from an all-gathered sample of 4096 keys per rank), every record travels once — grouped ncclSend /
 * ncclRecv — to the rank that owns its key range, and that rank runs the single-GPU post-processing (cmx_postprocess_gpu's
 * kernels) on what it received.  Duplicates agree in that key word, so a group never straddles two ranks.  Work per rank is
 * proportional to its share of the run, whereas cmx_dedup_exchange sorts the tuples of ALL ranks on every rank.
 * out_records / out_barcode_keys (capacity out_capacity, same kind of memory as the input): the records of THIS RANK'S KEY
 * RANGE in the reference's order, num_dups set, MAPQ-filtered, Tn5 applied (mapping_writer.h:254-287); the run's output is the
 * ranks' outputs one after the other in rank order.  CMX_ERR_INVALID with *n_out = the needed capacity if out_capacity is
 * too small (nothing is written then). */
typedef struct {
  float partition_ms, shuffle_ms, postprocess_ms; /* CUDA events on the context's stream */
  uint32_t n_ranks;
  uint64_t bytes_sent, bytes_received;            /* record bytes that left / reached this rank over NVLink */
  uint64_t n_received;                            /* records in this rank's key range before duplicate removal */
  uint64_t n_global;                              /* records of all ranks */
} cmx_shuffle_stats;
int cmx_dedup_shuffle(cmx_ctx *ctx, const void *records, const uint64_t *barcode_keys, uint64_t n, int on_device, void *out_records,
                      uint64_t *out_barcode_keys, uint64_t out_capacity, uint64_t *n_out, cmx_shuffle_stats *stats);
/* After the survivors of all ranks have been brought together (any transport; they are a small fraction of the run): the
 * reference's order and the deferred Tn5 shift (mapping_writer.h:285-287).  Host only (no device needed), in place. */
int cmx_exchange_finish(const cmx_params *params, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n);

#ifdef __cplusplus
}
#endif
#endif /* CHROMAP_B200_H_ */
