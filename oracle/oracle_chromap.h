// TEST INFRASTRUCTURE ONLY — CPU restatement ("oracle") of Chromap's per-read mapping hot path.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// build, link, import or execute anything under oracle/.  The product (chromap_b200/) never does.
//
// Parity pinning: this restatement is checked (tests/test_oracle_vs_reference.py, run in the build
// container where /root/reference exists) against the UNMODIFIED reference binary compiled by
// oracle/Makefile into oracle/_ref/chromap: BED output md5-identical on the reference's own
// test/ data (SURVEY.md §4 golden md5s) and on seeded synthetic data for --preset chip / atac.
// The reference ships no unit tests or golden vectors of its own (SURVEY.md §4), so the compiled
// binary is the only pin; the committed fixtures under tests/golden/ were produced by it.
//
// Every function cites the reference file:line it restates (paths relative to /root/reference/src).
#ifndef ORACLE_CHROMAP_H_
#define ORACLE_CHROMAP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

// Mirror of the MappingParameters fields used on the path (mapping_parameters.h:18-78).
typedef struct {
  int32_t error_threshold;        // -e, default 8
  int32_t min_num_seeds;          // -s, default 2
  int32_t max_seed_freq0;         // -f first, default 500
  int32_t max_seed_freq1;         // -f second, default 1000
  int32_t max_num_best_mappings;  // -n, default 1
  int32_t max_insert_size;        // -l, default 1000
  int32_t mapq_threshold;         // -q, default 30
  int32_t min_read_length;        // --min-read-length, default 30
  int32_t drop_repetitive_reads;  // default 500000
  int32_t trim_adapters;
  int32_t remove_pcr_duplicates;
  int32_t tn5_shift;
  int32_t split_alignment;
  int32_t low_memory_mode;
  int32_t output_format;  // 1 = BED, 5 = pairs (Hi-C, with split_alignment)
  int32_t single_end;     // records are single-end (MappingWithoutBarcode / MappingWithBarcode): changes duplicate equality and Tn5
} orc_params;

void orc_default_params(orc_params *p);
// preset: "chip" | "atac" | "hic" | "" (chromap_driver.cc:247-275).  Returns 0, or -1 if unknown.
int orc_apply_preset(orc_params *p, const char *preset);

typedef struct orc_index orc_index;
typedef struct orc_reference orc_reference;

// Index file loader (index.cc:132-169, khash.h:358-373) and builder (index.cc:12-89; the hash table
// layout differs from khash's insertion history but answers every lookup identically).
orc_index *orc_index_load(const char *path);
orc_index *orc_index_build(const orc_reference *ref, int k, int w);
int orc_index_save(const orc_index *idx, const char *path);
// From khash arrays in memory (copied), e.g. the arrays cmx_download_index() returns.
orc_index *orc_index_from_arrays(int k, int w, uint32_t n_buckets, const uint32_t *flags, const uint64_t *keys,
                                  const uint64_t *vals, const uint64_t *occ, uint32_t n_occ);
void orc_index_free(orc_index *idx);
int orc_index_k(const orc_index *idx);
int orc_index_w(const orc_index *idx);
// Raw views for uploading the same index to the device: khash arrays + occurrence table.
uint32_t orc_index_arrays(const orc_index *idx, const uint32_t **flags, const uint64_t **keys,
                          const uint64_t **vals, const uint64_t **occ, uint32_t *n_occ);
// kh_get + key/value fetch (khash.h:232-245).  Returns 1 if found.
int orc_index_lookup(const orc_index *idx, uint64_t minimizer_hash, uint64_t *key, uint64_t *val);

orc_reference *orc_reference_load(const char *fasta_path);
// Build from memory: n sequences, concatenated bases + offsets[n+1]; names may be NULL.
orc_reference *orc_reference_from_memory(uint32_t n, const char *concat, const uint64_t *offsets,
                                         const char *const *names);
void orc_reference_free(orc_reference *ref);
uint32_t orc_reference_num_sequences(const orc_reference *ref);
uint32_t orc_reference_length(const orc_reference *ref, uint32_t rid);
const char *orc_reference_name(const orc_reference *ref, uint32_t rid);
const char *orc_reference_seq(const orc_reference *ref, uint32_t rid);

// minimizer_generator.cc:7-139.  Writes up to cap (hash, hit) pairs; returns the count.
int orc_minimizers(const char *seq, uint32_t len, uint32_t seq_index, int k, int w, uint64_t *hash,
                   uint64_t *hit, int cap);

// alignment.cc:141-192 (scalar banded Myers).  pattern = reference window of read_len + 2e bytes.
int orc_banded_align(int e, const char *pattern, const char *text, int read_len, int *end_pos);
// alignment.cc:656-718.
void orc_banded_traceback(int e, int min_errors, const char *pattern, const char *text, int read_len,
                          int *start_pos);
int orc_align_dropoff(int e, const char *pattern, const char *text, int read_len, int from_3_end, int *end_pos, int *read_len_out);
// alignment.cc:24-83: extend an exact match into the skipped 5' gap of a split alignment (raw, signed char compares).
int orc_adjust_gap_beginning(int strand, const char *ref, const char *read, int *gap, int read_end, int ref_start, int ref_end);

// One PE record as emitted by mapping_generator.cc:110-123 (before sort/dedup).
typedef struct {
  uint32_t read_id;
  uint32_t rid;
  uint32_t fragment_start;
  uint16_t fragment_length;
  uint8_t mapq;
  uint8_t direction;  // 1 = read1 on + strand
  uint8_t is_unique;
  uint8_t num_dups;
  uint16_t positive_alignment_length;
  uint16_t negative_alignment_length;
} orc_pe_record;

// PairsMapping (pairs_mapping.h:11-49) without the read name: what --preset hic emits (mapping_generator.cc:169-210).
// Written into the same record buffer (24 bytes as well) when output_format == 5 (pairs).
typedef struct {
  uint32_t read_id;
  uint32_t rid1, rid2;
  uint32_t pos1, pos2;  // 0-based 5' positions, (rid1, pos1) <= (rid2, pos2)
  uint8_t strand1, strand2;  // 1 = +
  uint8_t mapq, is_unique;
} orc_pairs_record;

// Optional per-stage trace of one pair (for stage-level parity tests against the CUDA stages).
typedef struct {
  // per mate (index 0/1)
  int32_t n_minimizers[2];
  int32_t n_pos_candidates_gen[2], n_neg_candidates_gen[2];  // after GenerateCandidates
  int32_t n_pos_candidates[2], n_neg_candidates[2];          // entering verification
  int32_t n_pos_mappings[2], n_neg_mappings[2];
  int32_t min_errors[2], second_min_errors[2], n_best[2], n_second_best[2];
  uint32_t repetitive_seed_length[2];
  int32_t supplement_result;
  int32_t min_sum_errors, second_min_sum_errors, n_best_pairs, n_second_best_pairs;
  int32_t n_records;
  int32_t trimmed_len[2];
} orc_pair_trace;

typedef struct orc_mapper orc_mapper;  // params + borrowed index/reference
orc_mapper *orc_mapper_create(const orc_params *p, const orc_index *idx, const orc_reference *ref);
void orc_mapper_free(orc_mapper *m);

// The taskloop body, chromap.h:892-1143, for ONE reference batch: pairs [0, n) (n <= 500000 in the
// reference, chromap.h:182) given as concatenated ASCII + offsets.  Records are written to `out`
// (capacity cap_out) in read order; returns the number written.  first_read_id = running read counter
// (sequence_batch.cc:38-39).  trace may be NULL (else n entries).  Multi-mapper sampling restarts from
// mt19937(11) at every taskloop chunk (see orc_ref_task_chunks), exactly like the reference at any -t.
int64_t orc_map_pairs(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1,
                      const char *seq2, const uint32_t *off2, uint32_t first_read_id,
                      orc_pe_record *out, int64_t cap_out, orc_pair_trace *trace);
// Task chunks [starts[t], ends[t]) the reference's taskloop cuts pairs [0,n) into.  Returns #chunks.
int orc_ref_task_chunks(uint32_t n, uint32_t *starts, uint32_t *ends, int cap);
// Same as orc_map_pairs with chunks spread over n_threads host threads (results are identical).
int64_t orc_map_pairs_mt(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1,
                         const char *seq2, const uint32_t *off2, uint32_t first_read_id,
                         orc_pe_record *out, int64_t cap_out, int n_threads, orc_pair_trace *trace);

// ---- scATAC cell barcodes (chromap.cc:388-799): whitelist, abundance sampling, correction ------------------------
typedef struct orc_whitelist orc_whitelist;
orc_whitelist *orc_whitelist_load(const char *path, uint32_t bc_len);
void orc_whitelist_free(orc_whitelist *wl);
void orc_whitelist_sample(orc_whitelist *wl, const char *bcs, uint64_t n, uint32_t bc_len, uint64_t max_sample, uint32_t batch);
uint64_t orc_whitelist_arrays(const orc_whitelist *wl, const uint64_t **keys, const uint32_t **counts, uint64_t *num_sample);
void orc_mapper_set_barcodes(orc_mapper *m, const orc_whitelist *wl, int err_threshold, double prob_threshold, int output_not_in_whitelist);
int64_t orc_map_pairs_bc(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2, const uint32_t *off2,
                         const char *bcs, const char *quals, uint32_t bc_len, uint32_t first_read_id, orc_pe_record *out, uint64_t *out_bc,
                         int64_t cap_out, int n_threads, uint64_t *bc_stats);
int64_t orc_postprocess_bc(const orc_params *p, orc_pe_record *recs, uint64_t *bcs, int64_t n);
int64_t orc_format_bed_bc(const orc_reference *ref, const orc_pe_record *recs, const uint64_t *bcs, int64_t n, uint32_t bc_len, char *buf, int64_t cap);
int orc_run_files_bc(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                     const char *barcode_path, const char *whitelist_path, const char *out_path, int n_threads, uint64_t *bc_stats);

// Post-processing (mapping_processor.h:100-202, mapping_writer.h:166-376, chromap.h:1305-1355):
// sort / dedup / Tn5 / MAPQ filter, in place.  Returns the number of surviving records, sorted in
// output order (rid, then record operator<).
int64_t orc_postprocess(const orc_params *p, orc_pe_record *recs, int64_t n);
// Pairs post-processing (low-memory merge without dedup: sort by (rid1, rid2, pos1, pos2, mapq, read_id), MAPQ filter)
int64_t orc_postprocess_pairs(const orc_params *p, orc_pairs_record *recs, int64_t n);
// Pairs text with header (mapping_writer.cc:381-421); read_names[i] = name of read 1 of pair `read_id - first_read_id`.
int64_t orc_format_pairs(const orc_reference *ref, const orc_pairs_record *recs, int64_t n, const char *const *read_names,
                         uint32_t first_read_id, char *buf, int64_t cap);
// BED text (mapping_writer.cc:75-83).  Returns bytes written into buf (or needed if buf==NULL).
int64_t orc_format_bed(const orc_reference *ref, const orc_pe_record *recs, int64_t n, char *buf,
                       int64_t cap);

// Whole-file driver: FASTQ pair -> BED file, equivalent to `chromap -x idx -r ref -1 r1 -2 r2 -o out`.
int orc_run_files(const orc_params *p, const char *index_path, const char *ref_path,
                  const char *read1_path, const char *read2_path, const char *out_path,
                  int n_threads, double *mapping_seconds, uint64_t *n_pairs);


// Single-end (chromap.h:218-634 with MappingWithoutBarcode): records use orc_pe_record with both alignment lengths 0.
int64_t orc_map_reads_se(orc_mapper *m, uint32_t n, const char *seq, const uint32_t *off, uint32_t first_read_id, orc_pe_record *out,
                         int64_t cap_out, int n_threads);
int64_t orc_postprocess_se(const orc_params *p, orc_pe_record *recs, int64_t n);
int orc_run_files_se(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *out_path,
                     int n_threads);

int64_t orc_format_tagalign(const orc_reference *ref, const orc_pe_record *recs, int64_t n, char *buf, int64_t cap);

// Single-end reads with cell barcodes (MappingWithBarcode, bed_mapping.h:8-60); post-process with orc_postprocess_bc and single_end = 1.
int64_t orc_map_reads_se_bc(orc_mapper *m, uint32_t n, const char *seq, const uint32_t *off, const char *bcs, const char *quals, uint32_t bc_len,
                            uint32_t first_read_id, orc_pe_record *out, uint64_t *out_bc, int64_t cap_out, int n_threads, uint64_t *bc_stats);

// chromap --SAM for bulk reads, non-split (oracle only: groundwork for SURVEY.md 8f rank 3; read2_path NULL/"" = single-end).
int orc_run_files_sam(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                      const char *out_path);

// == cmx_sam_record
#define ORC_SAM_MAX_CIGAR 24
typedef struct {
  uint32_t read_id, rid;
  uint32_t pos[2], end[2];
  uint8_t strand[2];
  uint8_t mapq, is_unique, secondary;
  uint8_t n_cigar[2];
  uint8_t overflow;
  uint32_t cigar[2][ORC_SAM_MAX_CIGAR];
} orc_sam_record;
int64_t orc_map_sam_cores(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2, const uint32_t *off2, uint32_t first_read_id,
                          orc_sam_record *out, int64_t cap_out);
int orc_sg_align_test(const char *win, int wlen, const char *read, int rlen, int w, unsigned *cigar, int cap, int *start, int *end);

// chromap --PAF for bulk reads, non-split (oracle only: groundwork; the CUDA path does not emit PAF).
int orc_run_files_paf(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                      const char *out_path);

#ifdef __cplusplus
}
#endif
#endif  // ORACLE_CHROMAP_H_
