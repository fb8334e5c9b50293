// chromap_b200 — record sort / duplicate removal / MAPQ filter on the device (SURVEY.md §8f rank 1): the
// callers' side of the hot path.  Reference: the low-memory merge (mapping_writer.h:166-376), the in-memory
// sort + dedup (mapping_processor.h:100-202, chromap.h:1322-1355), operator< / operator== of the record types
// (bed_mapping.h:145-159,208-219, pairs_mapping.h:40-49).  Same results as the host routines in api.cu
// (cmx_postprocess / _bc / _pairs), which remain the specification the tests compare against.
//
// Order = the reference's total order on records, realised as an LSD radix sort over up to four 64-bit key
// words (CUB SortPairs is stable); the record index is the payload, records are gathered once at the end.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "device_common.cuh"

enum { PP_BED = 0, PP_BED_BC = 1, PP_PAIRS = 2, PP_BED_SE = 3 };  // PP_BED_SE: single-end records (MappingWithoutBarcode)

struct PpRecord {  // 24 bytes, viewed as cmx_pe_record or cmx_pairs_record
  u32 w[6];
};

struct PpParams {
  int kind, low_mem, dedup, tn5, mapq_threshold, se;
  int bulk = 0;  // PP_BED_BC with the low-memory rule: duplicates removed at bulk level (pp_bulk_* kernels)
};

// cmx_pe_record: w0 read_id, w1 rid, w2 fragment_start, w3 = fragment_length | mapq<<16 | direction<<24,
//                w4 = is_unique | num_dups<<8 | positive_alignment_length<<16, w5 = negative_alignment_length (low 16)
// cmx_pairs_record: w0 read_id, w1 rid1, w2 rid2, w3 pos1, w4 pos2, w5 = strand1 | strand2<<8 | mapq<<16 | is_unique<<24
__device__ __forceinline__ u32 pe_len(const PpRecord &r) { return r.w[3] & 0xFFFFu; }
__device__ __forceinline__ u32 pe_mapq(const PpRecord &r) { return (r.w[3] >> 16) & 0xFFu; }
__device__ __forceinline__ u32 pe_dir(const PpRecord &r) { return (r.w[3] >> 24) & 0xFFu; }
__device__ __forceinline__ u32 pe_uniq(const PpRecord &r) { return r.w[4] & 0xFFu; }
__device__ __forceinline__ u32 pe_pal(const PpRecord &r) { return r.w[4] >> 16; }
__device__ __forceinline__ u32 pe_nal(const PpRecord &r) { return r.w[5] & 0xFFFFu; }
__device__ __forceinline__ u32 pr_mapq(const PpRecord &r) { return (r.w[5] >> 16) & 0xFFu; }

// key word `word` (0 = most significant) of record r under the reference's order
__device__ __forceinline__ u64 pp_key_word(int kind, int word, const PpRecord &r, u64 bc) {
  if (kind == PP_PAIRS) {  // (rid1 bucket, rid2, pos1, pos2, mapq, read_id)
    if (word == 0) return ((u64)r.w[1] << 32) | r.w[2];
    if (word == 1) return ((u64)r.w[3] << 32) | r.w[4];
    return ((u64)pr_mapq(r) << 32) | r.w[0];
  }
  if (kind == PP_BED_BC) {  // (rid, start, length, barcode, mapq, direction, is_unique, read_id)
    if (word == 0) return ((u64)r.w[1] << 32) | r.w[2];
    if (word == 1) return (u64)pe_len(r);
    if (word == 2) return bc;
    return ((u64)((pe_mapq(r) << 16) | (pe_dir(r) << 8) | pe_uniq(r)) << 32) | r.w[0];
  }
  // (rid, start, length, mapq, direction, is_unique, read_id, positive length, negative length)
  if (word == 0) return ((u64)r.w[1] << 32) | r.w[2];
  if (word == 1) return ((u64)pe_len(r) << 48) | ((u64)pe_mapq(r) << 40) | ((u64)pe_dir(r) << 36) | ((u64)pe_uniq(r) << 32) | r.w[0];
  return ((u64)pe_pal(r) << 16) | pe_nal(r);
}
static inline int pp_n_words(int kind) { return kind == PP_BED_BC ? 4 : 3; }

__device__ __forceinline__ bool pp_same_fragment(int kind, int se, const PpRecord &a, u64 bca, const PpRecord &b, u64 bcb) {
  if (kind == PP_PAIRS) return a.w[1] == b.w[1] && a.w[2] == b.w[2] && a.w[3] == b.w[3] && a.w[4] == b.w[4];
  if (kind == PP_BED_SE) return a.w[1] == b.w[1] && a.w[2] == b.w[2];  // bed_mapping.h:89-92
  if (kind == PP_BED_BC && se) return a.w[1] == b.w[1] && a.w[2] == b.w[2] && bca == bcb;  // bed_mapping.h:36-39
  const bool s = a.w[1] == b.w[1] && a.w[2] == b.w[2] && pe_len(a) == pe_len(b);
  return kind == PP_BED_BC ? (s && bca == bcb) : s;
}

__device__ __forceinline__ void pp_tn5(PpRecord &r) {  // bed_mapping.h:225-230
  const u32 len = (pe_len(r) - 9u) & 0xFFFFu, pal = (pe_pal(r) - 4u) & 0xFFFFu, nal = (pe_nal(r) - 5u) & 0xFFFFu;
  r.w[2] += 4u;
  r.w[3] = (r.w[3] & 0xFFFF0000u) | len;
  r.w[4] = (r.w[4] & 0x0000FFFFu) | (pal << 16);
  r.w[5] = (r.w[5] & 0xFFFF0000u) | nal;
}

__device__ __forceinline__ void pp_tn5_se(PpRecord &r) {  // bed_mapping.h:97-103
  if (pe_dir(r) == 1u) r.w[2] += 4u;
  else r.w[3] = (r.w[3] & 0xFFFF0000u) | ((pe_len(r) - 5u) & 0xFFFFu);
}
__device__ __forceinline__ void pp_tn5_any(int kind, int se, PpRecord &r) { if (kind == PP_BED_SE || se) pp_tn5_se(r); else pp_tn5(r); }
__global__ void pp_tn5_kernel(int kind, int se, PpRecord *recs, u64 n) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pp_tn5_any(kind, se, recs[i]);
}
__global__ void pp_iota_kernel(u32 *idx, u64 n) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = (u32)i;
}
__global__ void pp_key_kernel(int kind, int word, const PpRecord *recs, const u64 *bcs, const u32 *idx, u64 n, u64 *keys) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u32 j = idx[i];
  keys[i] = pp_key_word(kind, word, recs[j], bcs ? bcs[j] : 0ull);
}
// largest value of key word 0 (the barcode plays no part in it): sizes the most significant radix passes
__global__ void pp_max_key0_kernel(int kind, const PpRecord *recs, u64 n, u64 *out) {
  u64 m = 0;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) m = max(m, pp_key_word(kind, 0, recs[i], 0ull));
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax((unsigned long long *)out, (unsigned long long)m);
}
__global__ void pp_gather_kernel(const PpRecord *recs, const u64 *bcs, const u32 *idx, u64 n, PpRecord *out, u64 *out_bc) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u32 j = idx[i];
  out[i] = recs[j];
  if (bcs) out_bc[i] = bcs[j];
}
__global__ void pp_head_kernel(int kind, int se, int dedup, const PpRecord *recs, const u64 *bcs, u64 n, u8 *head) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  head[i] = (!dedup || i == 0 || !pp_same_fragment(kind, se, recs[i - 1], bcs ? bcs[i - 1] : 0ull, recs[i], bcs ? bcs[i] : 0ull)) ? 1 : 0;
}
// One thread per run head: walks its run of equal fragments (runs are short: PCR duplicates), picks the survivor
// with the reference's rule, sets the duplicate count, applies the MAPQ filter and the deferred Tn5 shift.
// Out of place (recs -> res): nothing a thread reads is written by another.
__global__ void pp_resolve_kernel(PpParams P, const PpRecord *recs, const u64 *bcs, const u8 *head, u64 n, PpRecord *res, u64 *res_bc, u8 *keep_flag) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!head[i]) { keep_flag[i] = 0; return; }
  const int kind = P.kind;
  PpRecord keep = recs[i];
  u64 keep_bc = bcs ? bcs[i] : 0ull;
  u32 dups = 1;
  for (u64 j = i + 1; j < n && !head[j]; ++j) {
    const PpRecord r = recs[j];
    ++dups;
    if (kind == PP_PAIRS) { if (pr_mapq(r) > pr_mapq(keep)) keep = r; }                                      // mapping_writer.h:268-270
    else if (P.low_mem) { if (pe_mapq(r) > pe_mapq(keep)) { keep = r; keep_bc = bcs ? bcs[j] : 0ull; } }     // first of the highest MAPQ
    else { keep = r; keep_bc = bcs ? bcs[j] : 0ull; }                                                        // mapping_processor.h:181-197: the last
  }
  const u32 mq = kind == PP_PAIRS ? pr_mapq(keep) : pe_mapq(keep);
  const bool k = (int)mq >= P.mapq_threshold;
  if (k) {
    if (kind != PP_PAIRS) {
      if (P.dedup) keep.w[4] = (keep.w[4] & 0xFFFF00FFu) | ((dups > 255u ? 255u : dups) << 8);  // num_dups saturates (mapping_writer.h:282-284)
      if (P.low_mem && P.tn5) pp_tn5_any(kind, P.se, keep);
    }
    res[i] = keep;
    if (res_bc) res_bc[i] = keep_bc;
  }
  keep_flag[i] = k;
}

// ---------------------------------------------------------------------------------------------------------------
// Bulk-level duplicate removal of barcoded records (mapping_writer.h:126-163, 166-376), in place of pp_head_kernel and
// pp_resolve_kernel on the sorted records.  A bulk group is a run of records at the same position (rid, start, and length when
// paired-end); an entry is a run of consecutive records of one barcode inside a group.  An entry stands for its last record and
// weighs 1 (one record) or 2 (more: the merge overwrites the stored record, whose num_dups_ is 1, then adds 1).  A group keeps
// the record of its first entry with the greatest (weight, barcode abundance) and counts its records as duplicates.  No thread
// walks a group (scATAC hot spots hold 10^5 records and more): each entry tail gets a key whose maximum over the group, taken
// by CUB's reduce-by-key, names the survivor.
struct PpAbundance {  // the whitelist (cmx_upload_barcode_whitelist): barcode key -> count among the sampled barcodes
  const ulonglong2 *slots;
  u64 mask;
  int shift;
  unsigned long long *n_missing;  // += entries whose barcode is not in the table
  int top_listed;                 // the key ~0, kept out of the slots (wl_lookup)
  u64 top_count;
};
__device__ __forceinline__ bool pp_same_position(int se, const PpRecord &a, const PpRecord &b) {  // IsSamePosition, bed_mapping.h:43-45,155-158
  return a.w[1] == b.w[1] && a.w[2] == b.w[2] && (se || pe_len(a) == pe_len(b));
}
// head[i] = 1 at the first record of a bulk group.  key[i] = 0 inside an entry; at its last record
// (weight - 1) << 63 | abundance << 31 | (0x7FFFFFFF - i): the greatest key of a group is its first best entry (n < 2^31).
__global__ void pp_bulk_entry_kernel(int se, const PpRecord *recs, const u64 *bcs, u64 n, PpAbundance A, u32 *head, u64 *key) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  const u64 bc = bcs[i];
  const bool group_head = i == 0 || !pp_same_position(se, recs[i - 1], r);
  const bool entry_head = group_head || bcs[i - 1] != bc;
  const bool entry_tail = i + 1 == n || !pp_same_position(se, r, recs[i + 1]) || bcs[i + 1] != bc;
  head[i] = group_head ? 1u : 0u;
  u64 k = 0;
  if (entry_tail) {
    u64 abundance = 0;
    if (!wl_lookup(A.slots, A.mask, A.shift, A.top_listed, A.top_count, bc, &abundance)) atomicAdd(A.n_missing, 1ull);
    k = ((u64)!entry_head << 63) | ((abundance & 0xFFFFFFFFull) << 31) | (0x7FFFFFFFull - i);
  }
  key[i] = k;
}
// group_pos[g] = the first record of group g (gid = 1-based group of each record, the inclusive scan of head)
__global__ void pp_bulk_heads_kernel(const u32 *gid, u64 n, u32 *group_pos) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (i == 0 || gid[i] != gid[i - 1])) group_pos[gid[i] - 1] = (u32)i;
}
// *mapq = the highest MAPQ of the last group: the merge tests the last group's threshold on it (mapping_writer.h:323-337).
// Only records followed by a lower MAPQ (or by nothing) can hold it; inside a group they end runs of one length and barcode.
__global__ void pp_bulk_last_mapq_kernel(const PpRecord *recs, const u32 *group_pos, u32 n_groups, u64 n, unsigned *mapq) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i < group_pos[n_groups - 1]) return;
  const u32 mq = pe_mapq(recs[i]);
  if (i + 1 < n && pe_mapq(recs[i + 1]) >= mq) return;
  atomicMax(mapq, mq);
}
// One thread per group: its best entry's record with num_dups = min(255, group size), the MAPQ filter (the last group's on
// *last_mapq), Tn5.  Out of place (recs -> res[g]).
__global__ void pp_bulk_resolve_kernel(PpParams P, const PpRecord *recs, const u64 *bcs, const u64 *best, const u32 *group_pos, u32 n_groups, u64 n,
                                       const unsigned *last_mapq, PpRecord *res, u64 *res_bc, u8 *keep_flag) {
  const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const u32 b = 0x7FFFFFFFu - (u32)(best[g] & 0x7FFFFFFFull);
  const u32 dups = (u32)((g + 1 < n_groups ? (u64)group_pos[g + 1] : n) - group_pos[g]);
  PpRecord keep = recs[b];
  const u32 mq = g + 1 == n_groups ? *last_mapq : pe_mapq(keep);
  const bool k = (int)mq >= P.mapq_threshold;
  if (k) {
    keep.w[4] = (keep.w[4] & 0xFFFF00FFu) | ((dups > 255u ? 255u : dups) << 8);
    if (P.tn5) pp_tn5_any(P.kind, P.se, keep);
    res[g] = keep;
    res_bc[g] = bcs[b];
  }
  keep_flag[g] = k;
}

// ---------------------------------------------------------------------------------------------------------------
// Text writer on the device (SURVEY.md §8f rank 1): BED lines of mapping_writer.cc:75-83 (bulk: chrom start end N mapq
// strand dups) and :127-137 (barcoded: chrom start end barcode dups), byte-identical to cmx_format_bed[_bc].
// Pass 1 computes every line's length, an exclusive scan places the lines, pass 2 writes them.
__device__ __forceinline__ int dec_digits(u32 v) {
  int d = 1;
  while (v >= 10u) { v /= 10u; ++d; }
  return d;
}
__device__ __forceinline__ char *put_dec(char *p, u32 v) {  // writes v, returns the position after it
  const int d = dec_digits(v);
  for (int i = d - 1; i >= 0; --i) { p[i] = (char)('0' + v % 10u); v /= 10u; }
  return p + d;
}
// --barcode-translate on the device (cmx_upload_barcode_translation).  slots == nullptr: no table, the field is the barcode.
struct BedTranslation {
  const ulonglong2 *slots;  // {FROM key, TO offset << 16 | TO length}: kv_find's layout, as the whitelist's
  u64 mask;                 // n_slots - 1
  int shift;
  int from_len;             // L, 1..31
  const char *to;           // the TO strings
  unsigned long long *n_missing;  // length pass: += segments without an entry
  unsigned *first_missing;        // length pass: min over the launch's records i that have one
};
__global__ void tr_insert_kernel(const u64 *keys, const u64 *vals, u64 n, ulonglong2 *slots, u64 mask, int shift) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ulonglong2 *slot = kv_claim(slots, mask, shift, keys[i]);
  slot->y = vals[i];
}
// The barcode field of a barcoded line.  Without a table: the bc_len bases of the key (barcode_translator.h:114-123).  With
// one (Translate, barcode_translator.h:72-101): the TO strings of the key's nseg = bc_len / L segments joined by '-',
// segment s = the L bases that end (nseg - 1 - s) * L bases before the key's last, so the leading bc_len mod L bases play no
// part and nseg == 0 gives an empty field.  Writes to p unless it is nullptr; returns the field's length and adds the
// segments that have no entry to *n_missing (they contribute nothing).
__device__ __forceinline__ u32 bed_barcode_field(const BedTranslation &T, u64 bc, int bc_len, char *p, u32 *n_missing) {
  if (!T.slots) {
    if (p) for (int j = 0; j < bc_len; ++j) p[j] = "ACGT"[(bc >> ((bc_len - 1 - j) * 2)) & 3];
    return (u32)bc_len;
  }
  const int L = T.from_len, nseg = bc_len / L;
  const u64 seg_mask = (1ull << (2 * L)) - 1;
  u32 l = 0;
  for (int s = 0; s < nseg; ++s) {
    if (s) { if (p) p[l] = '-'; ++l; }
    u64 v;  // a FROM key has at most 31 bases, so it is never CMX_EMPTY_KEY (wl_lookup's case)
    if (!kv_find(T.slots, T.mask, T.shift, (bc >> (2 * L * (nseg - 1 - s))) & seg_mask, &v)) { ++*n_missing; continue; }
    const u32 tl = (u32)(v & 0xFFFFu);
    if (p) { const char *t = T.to + (v >> 16); for (u32 k = 0; k < tl; ++k) p[l + k] = t[k]; }
    l += tl;
  }
  return l;
}
__global__ void bed_len_kernel(const PpRecord *recs, u64 n, const u32 *name_off, int bc_len, u32 *len, const u64 *bcs = nullptr, BedTranslation T = {}) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  const u32 start = r.w[2], end = start + pe_len(r);
  const u32 nm = name_off[r.w[1] + 1] - name_off[r.w[1]];
  const u32 dups = (r.w[4] >> 8) & 0xFFu;
  u32 l = nm + 1 + dec_digits(start) + 1 + dec_digits(end) + 1;
  if (bc_len > 0) {
    u32 n_missing = 0;
    l += bed_barcode_field(T, T.slots ? bcs[i] : 0ull, bc_len, nullptr, &n_missing) + 1 + dec_digits(dups) + 1;
    if (n_missing) { atomicAdd(T.n_missing, (unsigned long long)n_missing); atomicMin(T.first_missing, (unsigned)i); }
  } else l += 1 + 1 + dec_digits(pe_mapq(r)) + 1 + 1 + 1 + dec_digits(dups) + 1;
  len[i] = l;
}
__global__ void bed_write_kernel(const PpRecord *recs, const u64 *bcs, u64 n, const char *names, const u32 *name_off, int bc_len,
                                 const u64 *off, u64 base, char *out, BedTranslation T = {}) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  char *p = out + (off[i] - base);
  const u32 a = name_off[r.w[1]], b = name_off[r.w[1] + 1];
  for (u32 k = a; k < b; ++k) *p++ = names[k];
  *p++ = '\t';
  p = put_dec(p, r.w[2]); *p++ = '\t';
  p = put_dec(p, r.w[2] + pe_len(r)); *p++ = '\t';
  const u32 dups = (r.w[4] >> 8) & 0xFFu;
  if (bc_len > 0) {
    u32 n_missing = 0;  // none: the length pass found every segment
    p += bed_barcode_field(T, bcs[i], bc_len, p, &n_missing);
    *p++ = '\t';
  } else {
    *p++ = 'N'; *p++ = '\t';
    p = put_dec(p, pe_mapq(r)); *p++ = '\t';
    *p++ = pe_dir(r) ? '+' : '-'; *p++ = '\t';
  }
  p = put_dec(p, dups);
  *p++ = '\n';
}

// pairs lines of mapping_writer.cc:405-421: readID chrom1 pos1 chrom2 pos2 strand1 strand2 UU mapq mapq (1-based positions)
__global__ void pairs_len_kernel(const PpRecord *recs, u64 n, const u32 *name_off, const u64 *rname_off, u32 first_read_id, u32 *len) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  const u32 ri = r.w[0] - first_read_id;
  const u32 mq = pr_mapq(r);
  len[i] = (u32)(rname_off[ri + 1] - rname_off[ri]) + 1 + (name_off[r.w[1] + 1] - name_off[r.w[1]]) + 1 + dec_digits(r.w[3] + 1u) + 1 +
           (name_off[r.w[2] + 1] - name_off[r.w[2]]) + 1 + dec_digits(r.w[4] + 1u) + 1 + 2 + 2 + 3 + dec_digits(mq) + 1 + dec_digits(mq) + 1;
}
__global__ void pairs_write_kernel(const PpRecord *recs, u64 n, const char *names, const u32 *name_off, const char *rnames, const u64 *rname_off,
                                   u32 first_read_id, const u64 *off, char *out) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  char *p = out + off[i];
  const u32 ri = r.w[0] - first_read_id;
  for (u64 k = rname_off[ri]; k < rname_off[ri + 1]; ++k) *p++ = rnames[k];
  *p++ = '\t';
  for (u32 k = name_off[r.w[1]]; k < name_off[r.w[1] + 1]; ++k) *p++ = names[k];
  *p++ = '\t';
  p = put_dec(p, r.w[3] + 1u); *p++ = '\t';
  for (u32 k = name_off[r.w[2]]; k < name_off[r.w[2] + 1]; ++k) *p++ = names[k];
  *p++ = '\t';
  p = put_dec(p, r.w[4] + 1u); *p++ = '\t';
  *p++ = (r.w[5] & 0xFFu) ? '+' : '-'; *p++ = '\t';
  *p++ = ((r.w[5] >> 8) & 0xFFu) ? '+' : '-'; *p++ = '\t';
  *p++ = 'U'; *p++ = 'U'; *p++ = '\t';
  const u32 mq = pr_mapq(r);
  p = put_dec(p, mq); *p++ = '\t';
  p = put_dec(p, mq); *p++ = '\n';
}
