// chromap_b200 — SAM coordinates and CIGARs on the device (SURVEY.md §8f rank 3): per REPORTED mapping the reference
// replaces BandedTraceback by ksw_semi_global3 (ksw.cc:505-626: semi-global affine DP of the read against the
// verification window, band 2e+1, one direction byte per cell, traceback) when the output is SAM
// (mapping_generator.h:723-760,807-855); coordinates, alignment lengths and therefore MAPQ follow from it.
// The device writes fixed-size cores (positions, strands, MAPQ, CIGARs); NM / MD and the text are host work over
// the CIGAR (cmx_format_sam), like the reference's writer.
#pragma once
#ifdef __CUDACC__
#include "device_common.cuh"
#endif

#define SAM_MAX_L 160                 // the short instance: reads up to 160 bases (2 x 150 bp fits)
#define SAM_MAX_L_LONG 320            // the long instance, for contexts sized above 160 bases; longer reads are reported, not aligned
#define SAM_MAX_E 8                   // -e up to 8 (every preset that writes SAM); keeps the per-thread direction matrix at 18 x MaxL bytes
#define SAM_MAX_CIGAR 24              // == CMX_SAM_MAX_CIGAR

#ifdef __CUDACC__
#define SAM_HD __host__ __device__ __forceinline__
#else
#define SAM_HD inline
#endif

// Semi-global affine alignment of the read against its verification window with the scores and tie rules of
// ksw_semi_global3 (ksw.cc:505-626), for the one shape the SAM path uses it in (mapping_generator.h:723-760, 807-855):
// window = read length + 2e, band w = 2e + 1, the read may start anywhere in the first w window positions for free.
//
// Formulated on DIAGONALS instead of columns: cell (i, j) of the band is (i, d = j - i), d = 0 .. w.  The three inputs of a
// cell then sit at fixed places — the diagonal predecessor at the same d of the previous row, the vertical gap state at
// d + 1 of the previous row, the horizontal gap state at d - 1 of this row — so the whole band state is two small arrays of
// w + 2 integers that are updated in place and live in registers (the loop over d is unrolled; e <= 8 gives 18 cells),
// and a row touches nothing else but its w + 1 direction bytes.  No per-column score arrays, no row buffers.
//   m = diagonal + score;  h = max(m, e, f) with ties to m, then to the larger of (m, e) over f;
//   e' = max(e - e_del, m - (o_del + e_del)), f' = max(f - e_ins, m - (o_ins + e_ins)), the "continue the gap" bit set only
//   when strictly larger (ksw's rule: gaps open from m, not from h).
// Direction byte: bits 0-1 the source of h (0 diagonal, 1 vertical, 2 horizontal), bits 2-3 / 4-5 the gap continuation
// states, read back by the traceback exactly as ksw does.  WIN(j): base code of the window at j, RD(i): base code of the
// read at i; scores: match / -mismatch between codes < 4, 0 if either is "other" (mapping_generator.h:661-670).
// Returns the number of CIGAR operations (BAM encoding len << 4 | op, M = 0, I = 1, D = 2) or -1 if they do not fit `cap`.
// MaxL: the longest read the direction matrix holds (rlen <= MaxL); it lives in local memory, 18 x MaxL bytes per thread.
#define SAM_BAND (2 * SAM_MAX_E + 2)  // cells per row
template <int MaxL = SAM_MAX_L, typename WinF, typename ReadF>
SAM_HD int sam_band_align(int rlen, int e, int match, int mismatch, int o_del, int e_del, int o_ins, int e_ins, WinF WIN, ReadF RD, unsigned int *cigar, int cap,
                          int *start, int *end) {
  const int NEG = -0x40000000;
  const int w = 2 * e + 1, wlen = rlen + 2 * e;
  const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
  int hd[SAM_BAND], ed[SAM_BAND + 1];
  unsigned char dirs[SAM_BAND * MaxL];
#pragma unroll
  for (int d = 0; d < SAM_BAND; ++d) { hd[d] = 0; ed[d] = NEG; }  // free start on every diagonal of the band
  ed[SAM_BAND] = NEG;
  for (int i = 0; i < rlen; ++i) {
    const unsigned int rc = RD(i);
    unsigned char *row = &dirs[i * (w + 1)];
    int f = NEG;
#pragma unroll
    for (int d = 0; d < SAM_BAND; ++d) {
      if (d > w || i + d >= wlen) break;
      const unsigned int wc = WIN(i + d);
      const int m = hd[d] + ((rc < 4u && wc < 4u) ? (rc == wc ? match : -mismatch) : 0);
      int ev = d < w ? ed[d + 1] : NEG;  // the cell above lies outside the previous row's band on the last diagonal
      unsigned char dir = m >= ev ? 0 : 1;
      int h = m >= ev ? m : ev;
      if (!(h >= f)) { dir = 2; h = f; }
      hd[d] = h;
      const int td = m - oe_del, ti = m - oe_ins;
      ev -= e_del;
      if (ev > td) dir |= 1 << 2; else ev = td;
      ed[d] = ev;
      f -= e_ins;
      if (f > ti) dir |= 2 << 4; else f = ti;
      row[d] = dir;
    }
  }
  // the read ends on the last row: best of the last w window positions, the rightmost first (ksw.cc:585-590)
  int score = hd[w - 1], best = wlen;
  for (int j = 1; j < w; ++j) if (hd[w - 1 - j] > score) { score = hd[w - 1 - j]; best = wlen - j; }
  *end = best;
  // traceback from (rlen - 1, best - 1): operations come out last to first, equal neighbours merged
  int n = 0, i = rlen - 1, k = best - 1, which = 0;
  bool ovf = false;
  auto push = [&](unsigned int op, unsigned int len) {
    if (n > 0 && (cigar[n - 1] & 0xfu) == op) cigar[n - 1] += len << 4;
    else if (n < cap) cigar[n++] = (len << 4) | op;
    else ovf = true;
  };
  while (i >= 0 && k >= 0) {
    which = dirs[i * (w + 1) + (k - i)] >> (which << 1) & 3;
    if (which == 0) { push(0u, 1u); --i; --k; }
    else if (which == 1) { push(1u, 1u); --i; }
    else { push(2u, 1u); --k; }
  }
  if (i >= 0) push(1u, (unsigned int)(i + 1));
  *start = k + 1;
  if (ovf) return -1;
  for (int a = 0, b = n - 1; a < b; ++a, --b) { const unsigned int t = cigar[a]; cigar[a] = cigar[b]; cigar[b] = t; }
  return n;
}

#if defined(__CUDACC__) || defined(CMX_HOST_EMU)
struct OutSam {  // == cmx_sam_record
  u32 read_id, rid;
  u32 pos[2], end[2];  // 0-based inclusive reference span of mate 1 / mate 2 (single-end: index 0)
  u8 strand[2];        // 1 = +
  u8 mapq, is_unique, secondary;
  u8 n_cigar[2];
  u8 overflow;         // read longer than the instance's MaxL or CIGAR longer than SAM_MAX_CIGAR: reported, not written
  u32 cigar[2][SAM_MAX_CIGAR];
};

// SAM branch of GetRefStartEndPositionForReadFromMapping, non-split (mapping_generator.h:696-760 for the + strand,
// :807-855 for the - strand: same call on the reverse complement with read_start_site = 0).  Returns false on overflow.
template <int MaxL>
__device__ __noinline__ bool sam_span(const DevParams &P, const DevRef &R, const u8 *read, int L, int strand, u64 dpos, u32 *st, u32 *en, u32 *cigar,
                                         u8 *n_cigar) {
  const int e = P.e;
  const u32 rid = (u32)(dpos >> 32), rp = (u32)dpos;
  u32 vws = rp + 1u > (u32)(L + e) ? rp + 1u - (u32)L - (u32)e : 0u;
  if (rp + (u32)e >= R.len[rid]) vws = R.len[rid] - (u32)e - (u32)L;
  *st = vws; *en = vws; *n_cigar = 0;
  if (L > MaxL || e > SAM_MAX_E) return false;
  const u8 *win = R.seq + R.off[rid] + vws;
  int s0 = 0, e0 = 0, n;
  if (strand == 0)
    n = sam_band_align<MaxL>(L, e, 1, 4, 6, 1, 6, 1, [&](int j) { return base_code(__ldg(win + j)); }, [&](int i) { return base_code(read[i]); }, cigar, SAM_MAX_CIGAR, &s0,
                       &e0);
  else
    n = sam_band_align<MaxL>(L, e, 1, 4, 6, 1, 6, 1, [&](int j) { return base_code(__ldg(win + j)); }, [&](int i) { return neg_code(read, L, i); }, cigar, SAM_MAX_CIGAR, &s0,
                       &e0);
  *st = vws + (u32)s0;
  *en = vws + (u32)e0 - 1u;
  if (n < 0) return false;
  *n_cigar = (u8)n;
  return true;
}

// emit_kernel with the SAM span: ProcessBestMappingsForPairedEndReadOnOneDirection (mapping_generator.h:486-654) + the fields
// EmplaceBackPairedEndMappingRecord<SAMMapping> needs (mapping_generator.cc:84-107); flags and TLEN are derived on the host.
template <int MaxL>
__global__ void emit_sam_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutSam *out, int *out_n, Counters *ctr) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status == ST_OVERFLOW) return;
  if (pm.status != ST_OK || pm.n_best > P.drop_rep || pm.n_best == 0) { out_n[pair] = 0; return; }
  const ReadMeta *rm = S.rmeta + 2 * slot;
  const int mb = P.max_best;
  const int to_report = mb < pm.n_best ? mb : pm.n_best;
  const int *sel = pair_sel + (size_t)pair * mb;
  const u8 uniq = (pm.n_best == 1 || rm[0].n_best == 1 || rm[1].n_best == 1) ? 1 : 0;
  const int force = pm.sup != 0 ? 0 : -1;
  int idx = 0, reported = 0;
  const int L[2] = {rm[0].len, rm[1].len};
  const u8 *rd[2] = {read_ptr(B, pair, 0), read_ptr(B, pair, 1)};
  for (int dir = 0; dir < 2 && reported != to_report; ++dir) {
    const int s1 = dir, s2 = 1 - dir;
    const Strided<u64> p1 = map_pos_of(S, 2 * slot, s1), p2 = map_pos_of(S, 2 * slot + 1, s2);
    const Strided<short> e1 = map_err_of(S, 2 * slot, s1), e2 = map_err_of(S, 2 * slot + 1, s2);
    pair_sweep_until(P, s1, (u32)L[0], (u32)L[1], p1, e1, rm[0].n_map[s1], p2, e2, rm[1].n_map[s2], [&](int i1, int j, int sum) -> bool {
      if (sum != pm.min_sum) return false;
      if (idx == sel[reported]) {
        OutSam &o = out[(size_t)pair * mb + reported];
        u32 st1, en1, st2, en2;
        const bool ok1 = sam_span<MaxL>(P, R, rd[0], L[0], s1, p1[i1], &st1, &en1, o.cigar[0], &o.n_cigar[0]);
        const bool ok2 = sam_span<MaxL>(P, R, rd[1], L[1], s2, p2[j], &st2, &en2, o.cigar[1], &o.n_cigar[1]);
        const unsigned short al1 = (unsigned short)(en1 - st1 + 1u), al2 = (unsigned short)(en2 - st2 + 1u);
        o.read_id = B.first_read_id + (u32)pair;
        o.rid = (u32)(p1[i1] >> 32);
        o.pos[0] = st1; o.end[0] = en1; o.pos[1] = st2; o.end[1] = en2;
        o.strand[0] = s1 == 0 ? 1 : 0; o.strand[1] = s2 == 0 ? 1 : 0;
        o.mapq = mapq_pe(T, e1[i1], e2[j], al1, al2, L[0], L[1], force, pm, rm);
        o.is_unique = uniq;
        o.secondary = reported >= 1 ? 1 : 0;
        o.overflow = (ok1 && ok2) ? 0 : 1;
        if (o.overflow) agg_add(&ctr->n_overflow, 1ull);
        ++reported;
      }
      ++idx;
      return reported == to_report;
    });
  }
  out_n[pair] = reported;
  pm.n_rec = reported;
  if (reported > 0) { agg_add(&ctr->n_mapped, 1ull); if (pm.n_best == 1) agg_add(&ctr->n_unique, 1ull); }
}

// emit_se_kernel with the SAM span (mapping_generator.h:256-343 with MAPPINGFORMAT_SAM)
template <int MaxL>
__global__ void emit_sam_se_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutSam *out, int *out_n, Counters *ctr) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status == ST_OVERFLOW) return;
  if (pm.status != ST_OK || pm.n_best == 0) { out_n[pair] = 0; return; }
  const ReadMeta &rm = S.rmeta[2 * slot];
  const int mb = P.max_best, e = P.e, L = rm.len;
  const int to_report = mb < rm.n_best ? mb : rm.n_best;
  const int *sel = pair_sel + (size_t)pair * mb;
  const u8 *r = read_ptr(B, pair, 0);
  int idx = 0, reported = 0;
  for (int s = 0; s < 2 && reported != to_report; ++s) {
    const Strided<u64> mp = map_pos_of(S, 2 * slot, s);
    const Strided<short> me = map_err_of(S, 2 * slot, s);
    for (int mi = 0; mi < rm.n_map[s]; ++mi) {
      if ((int)me[mi] > rm.min_err) continue;
      if (idx == sel[reported]) {
        OutSam &o = out[(size_t)pair * mb + reported];
        u32 st, en;
        const bool ok = sam_span<MaxL>(P, R, r, L, s, mp[mi], &st, &en, o.cigar[0], &o.n_cigar[0]);
        const unsigned short al = (unsigned short)(en - st + 1u);
        o.read_id = B.first_read_id + (u32)pair;
        o.rid = (u32)(mp[mi] >> 32);
        o.pos[0] = st; o.end[0] = en; o.pos[1] = 0; o.end[1] = 0;
        o.strand[0] = s == 0 ? 1 : 0; o.strand[1] = 0;
        o.mapq = mapq_se(T, (int)me[mi], al, L, e, rm);
        o.is_unique = rm.n_best == 1 ? 1 : 0;
        o.secondary = reported >= 1 ? 1 : 0;
        o.n_cigar[1] = 0;
        o.overflow = ok ? 0 : 1;
        if (o.overflow) agg_add(&ctr->n_overflow, 1ull);
        if (++reported == to_report) break;
      }
      ++idx;
    }
  }
  out_n[pair] = reported;
  pm.n_rec = reported;
  if (reported > 0) { agg_add(&ctr->n_mapped, 1ull); if (rm.n_best == 1) agg_add(&ctr->n_unique, 1ull); }
}

// read-order compaction of records of any size (whole 4-byte words)
__global__ void compact_words_kernel(int n_pairs, int mb, int rec_words, const u32 *in, const int *n_rec, const u64 *offs, u32 *out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  const int n = n_rec[p];
  const u32 *src = in + (size_t)p * mb * rec_words;
  u32 *dst = out + (size_t)offs[p] * rec_words;
  for (int i = 0; i < n * rec_words; ++i) dst[i] = src[i];
}
#endif
