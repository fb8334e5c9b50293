// chromap_b200 — FASTQ text -> packed read batch on the device (SURVEY.md §8f rank 1): the loader side of the hot
// path.  Replaces, for 4-line FASTQ, SequenceBatch::LoadBatch + kseq_read (sequence_batch.cc:9-60, kseq.h:177-222):
// name = header after '@' up to the first whitespace, sequence / quality lines with '\n' (and a trailing '\r') stripped,
// every other byte kept as it is.  Multi-line records, FASTA reads and empty reads are reported, not guessed at
// (the caller then uses its host parser).
#pragma once
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "device_common.cuh"

__global__ void newline_flag_kernel(const char *text, u32 n, u8 *flag) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = text[i] == '\n' ? 1 : 0;
}

struct IngestStats {  // device-side summary of one chunk
  u32 bad_header, bad_plus, empty_reads, qual_mismatch, min_len, max_len;
};

// one thread per record: the five newline positions around it -> sequence / quality spans, name span, checks
__global__ void ingest_record_kernel(const char *text, const u32 *nl, u32 n_rec, u32 *seq_start, u32 *qual_start, u32 *len, u32 *spans, IngestStats *st) {
  const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rec) return;
  const u32 h0 = r == 0 ? 0u : nl[4 * r - 1] + 1u;  // header line start
  const u32 h1 = nl[4 * r];                          // header line end ('\n')
  const u32 s1 = nl[4 * r + 1], p1 = nl[4 * r + 2], q1 = nl[4 * r + 3];
  u32 sl = s1 - (h1 + 1u), ql = q1 - (p1 + 1u);
  if (sl > 0 && text[s1 - 1] == '\r') --sl;
  if (ql > 0 && text[q1 - 1] == '\r') --ql;
  if (text[h0] != '@') atomicAdd(&st->bad_header, 1u);
  if (text[s1 + 1] != '+') atomicAdd(&st->bad_plus, 1u);
  if (sl == 0) atomicAdd(&st->empty_reads, 1u);
  if (ql != sl) atomicAdd(&st->qual_mismatch, 1u);
  atomicMin(&st->min_len, sl);
  atomicMax(&st->max_len, sl);
  seq_start[r] = h1 + 1u; qual_start[r] = p1 + 1u; len[r] = sl;
  if (spans) {  // kseq: the name ends at the first whitespace of the header
    u32 e = h0 + 1u;
    while (e < h1 && !(text[e] == ' ' || text[e] == '\t' || text[e] == '\r')) ++e;
    spans[2 * r] = h0 + 1u; spans[2 * r + 1] = e - (h0 + 1u);
  }
}
// one warp per record: copy its bases (and qualities) to their packed place
// (a record whose quality line is shorter than its sequence is reported by ingest_record_kernel; the copy here never
// leaves the quality line, so such a chunk cannot read past the text or write past the packed buffers)
__global__ void ingest_pack_kernel(const char *text, const u32 *seq_start, const u32 *qual_start, const u32 *off, const u32 *nl, u32 n_rec, char *seq,
                                   char *qual) {
  const u32 r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= n_rec) return;
  const u32 o = off[r], l = off[r + 1] - o, s = seq_start[r];
  for (u32 i = lane; i < l; i += 32) seq[o + i] = text[s + i];
  if (qual) {
    const u32 q = qual_start[r], ql = min(l, nl[4 * r + 3] - q);
    for (u32 i = lane; i < ql; i += 32) qual[o + i] = text[q + i];
  }
}

// --read-format (sequence_effective_range.h:80-118) on the same records: a length pass between ingest_record_kernel and the
// offset scan, and a pack kernel in ingest_pack_kernel's place.
#define CUT_MAX_RANGES 8
struct CutRanges {  // cmx_read_range as the kernels take it: ranges ascending and disjoint, end == -1 in the last one only
  u32 n;
  int start[CUT_MAX_RANGES], end[CUT_MAX_RANGES];
  int reverse;
};
struct CutStats {  // device-side summary of the cut
  u32 out_of_range, empty, min_len, max_len;
};

// one thread per record: raw length -> cut length, in place.  A record whose read ends before an explicit range end gets
// length 0 (nothing is packed for it) and is counted; so is a record with nothing left after the cut.
__global__ void ingest_cut_len_kernel(u32 *len, u32 n_rec, CutRanges range, CutStats *st) {
  const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rec) return;
  const u32 l = len[r];
  u32 c = 0;
  bool over = false;
#pragma unroll
  for (u32 k = 0; k < CUT_MAX_RANGES; ++k) {  // unrolled: constant indices keep the ranges in registers
    if (k >= range.n) break;
    const u32 a = (u32)range.start[k];
    if (range.end[k] == -1) c += l > a ? l - a : 0u;  // the last range only
    else {
      over |= (u32)range.end[k] >= l;
      c += (u32)range.end[k] - a + 1u;
    }
  }
  if (over) { atomicAdd(&st->out_of_range, 1u); c = 0; }
  else if (c == 0) atomicAdd(&st->empty, 1u);
  atomicMin(&st->min_len, c);
  atomicMax(&st->max_len, c);
  len[r] = c;
}

// ACGTacgt -> the upper-case complement, every other byte -> 'N' (utils.h:87-100)
struct CutComplement {
  u8 c[256];
};
constexpr CutComplement make_cut_complement() {
  CutComplement t{};
  for (int i = 0; i < 256; ++i) t.c[i] = 'N';
  t.c['A'] = t.c['a'] = 'T'; t.c['C'] = t.c['c'] = 'G'; t.c['G'] = t.c['g'] = 'C'; t.c['T'] = t.c['t'] = 'A';
  return t;
}
__device__ const CutComplement kCutComplement = make_cut_complement();

// one warp per record: gather the bases (and qualities) of its ranges straight from the text to their packed place; with
// range.reverse the bases are complemented and both are written back to front.  Reads and writes of a warp are consecutive
// bytes either way.  The quality copy stays inside the quality line (see ingest_pack_kernel).
__global__ void ingest_cut_pack_kernel(const char *text, const u32 *seq_start, const u32 *qual_start, const u32 *off, const u32 *nl, u32 n_rec,
                                       CutRanges range, char *seq, char *qual) {
  const u32 r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= n_rec) return;
  const u32 o = off[r], l = off[r + 1] - o, s = seq_start[r];
  const u32 q = qual ? qual_start[r] : 0u, qe = qual ? nl[4 * r + 3] - q : 0u;
  const bool rev = range.reverse != 0;
  u32 done = 0;  // bases of the cut before range k
  for (u32 k = 0; k < range.n && done < l; ++k) {
    const u32 a = (u32)range.start[k];
    const u32 m = range.end[k] == -1 ? l - done : min(l - done, (u32)range.end[k] - a + 1u);
    for (u32 i = lane; i < m; i += 32) {
      const u32 dst = o + (rev ? l - 1u - (done + i) : done + i);
      const u8 b = (u8)text[s + a + i];
      seq[dst] = rev ? (char)kCutComplement.c[b] : (char)b;
      if (qual && a + i < qe) qual[dst] = text[q + a + i];
    }
    done += m;
  }
}
