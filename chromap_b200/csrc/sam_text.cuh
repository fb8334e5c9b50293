// chromap_b200 — SAM text on the device, byte-identical to cmx_format_sam_bc / cmx_format_sam (host/sam_writer.cc, which stays
// the specification).  From the SAM cores: one line per mate (flags, mate fields and TLEN of mapping_generator.h:613-640), the
// order of SAMMapping::operator< with the cell barcode (sam_mapping.h:188-193) as stable LSD radix passes over line ids, runs
// of SAMMapping::operator== (:194-199) resolved to their survivor (in memory the last, mapping_processor.h:181-197; low memory
// the first of the highest MAPQ, mapping_writer.h:268-270), the MAPQ filter, then the lines of mapping_writer.cc:324-356 with
// NM / MD (alignment.cc:85-139) and CB:Z: (:350-354) in a length pass, an exclusive scan and a write pass.
//
// A line id is 2 * core + mate (paired-end) or the core (single-end), so ascending ids are the order the host writer expands
// the cores in and the radix passes keep ties in it, as its std::stable_sort does.
#pragma once
#include "postprocess.cuh"
#include "sam_kernels.cuh"

struct SamReads {          // one read file's reads first_read_id .. on the device
  const char *seq, *qual;  // qual == nullptr: QUAL is empty
  const u64 *off;          // [n + 1] into seq / qual
  const char *names;
  const u64 *name_off;     // [n + 1] into names
};
struct SamText {
  const OutSam *cores;
  const u64 *bcs;            // cell barcode key per core; nullptr: bulk (no CB tag, barcode 0 in the order)
  int pe, bc_len;
  u32 first_read_id;
  SamReads r[2];             // mate 1 / mate 2 (single-end: r[0])
  const u8 *ref;             // the reference as cmx_upload_reference laid it out
  const u64 *ref_off;
  const char *ref_names;
  const u32 *ref_name_off;   // [n_seq + 1] into ref_names
};

struct SamLine {
  u32 core, rid, pos, mpos, read_id;
  int mate, mrid, flag, tlen, mapq;
};
__device__ __forceinline__ SamLine sam_line(const SamText &T, u32 l) {
  SamLine s;
  s.core = T.pe ? l >> 1 : l;
  s.mate = T.pe ? (int)(l & 1u) : 0;
  const OutSam &c = T.cores[s.core];
  s.rid = c.rid; s.read_id = c.read_id; s.mapq = c.mapq;
  s.pos = c.pos[s.mate];
  if (!T.pe) {
    s.mpos = 0; s.mrid = -1; s.tlen = 0;
    s.flag = (c.strand[0] ? 0 : 16) | (c.secondary ? 256 : 0);
    return s;
  }
  int f = s.mate ? (3 | 128) : (3 | 64);
  if (!c.strand[0]) f |= s.mate ? 32 : 16;
  if (!c.strand[1]) f |= s.mate ? 16 : 32;
  if (c.secondary) f |= 256;
  const int tlen = c.strand[0] ? (int)(c.end[1] - c.pos[0] + 1u) : (int)(c.end[0] - c.pos[1] + 1u);  // GetFragmentLength
  s.flag = f;
  s.mpos = c.pos[1 - s.mate]; s.mrid = (int)c.rid;
  s.tlen = c.strand[s.mate] ? tlen : -tlen;
  return s;
}
__device__ __forceinline__ u64 sam_bc(const SamText &T, const SamLine &s) { return T.bcs ? T.bcs[s.core] : 0ull; }

// key word `word` (0 = most significant) of line l: (rid, pos), barcode, mate position, (read 1, mapq, read id).  The mate's
// rid is the line's own rid or -1 for every line of a call, so word 0 decides it.
__device__ __forceinline__ u64 sam_key_word(const SamText &T, int word, u32 l) {
  const SamLine s = sam_line(T, l);
  if (word == 0) return ((u64)s.rid << 32) | s.pos;
  if (word == 1) return sam_bc(T, s);
  if (word == 2) return s.mpos;
  return ((u64)((s.flag >> 6) & 1) << 40) | ((u64)s.mapq << 32) | s.read_id;
}
// identity ids, the largest key word 0 (sizes its radix pass) and the overflowed cores' lines (err[0])
__global__ void sam_expand_kernel(SamText T, u64 n_lines, u32 *idx, u64 *max0, int *err) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u64 k = 0;
  if (i < n_lines) {
    idx[i] = (u32)i;
    k = sam_key_word(T, 0, (u32)i);
    if (T.cores[T.pe ? i >> 1 : i].overflow) atomicAdd(err, 1);
  }
  for (int o = 16; o; o >>= 1) k = max(k, __shfl_xor_sync(0xffffffffu, k, o));
  if ((threadIdx.x & 31) == 0 && k) atomicMax((unsigned long long *)max0, (unsigned long long)k);
}
// the largest read index (read id - first_read_id) of the cores: how many reads of each file the call needs
__global__ void sam_max_read_kernel(SamText T, u64 n_lines, u32 *max_ri) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u32 r = 0;
  if (i < n_lines) r = T.cores[T.pe ? i >> 1 : i].read_id - T.first_read_id;
  for (int o = 16; o; o >>= 1) r = max(r, __shfl_xor_sync(0xffffffffu, r, o));
  if ((threadIdx.x & 31) == 0 && r) atomicMax(max_ri, r);
}
__global__ void sam_key_kernel(SamText T, int word, const u32 *idx, u64 n, u64 *keys) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = sam_key_word(T, word, idx[i]);
}
__device__ __forceinline__ bool sam_same(const SamText &T, u32 a, u32 b) {  // operator==: (pos, rid, barcode, read 1, mrid, mpos)
  const SamLine x = sam_line(T, a), y = sam_line(T, b);
  return x.pos == y.pos && x.rid == y.rid && sam_bc(T, x) == sam_bc(T, y) && ((x.flag ^ y.flag) & 64) == 0 && x.mrid == y.mrid && x.mpos == y.mpos;
}
__global__ void sam_head_kernel(SamText T, int dedup, const u32 *idx, u64 n, u8 *head) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = (!dedup || i == 0 || !sam_same(T, idx[i - 1], idx[i])) ? 1 : 0;
}
// one thread per run head: the survivor's line id in res[i], keep[i] = it passes the MAPQ filter
__global__ void sam_resolve_kernel(SamText T, int low_mem, int mapq_threshold, const u32 *idx, const u8 *head, u64 n, u32 *res, u8 *keep) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!head[i]) { keep[i] = 0; return; }
  u32 k = idx[i];
  int kq = T.cores[T.pe ? k >> 1 : k].mapq;
  for (u64 j = i + 1; j < n && !head[j]; ++j) {
    const u32 l = idx[j];
    const int q = T.cores[T.pe ? l >> 1 : l].mapq;
    if (!low_mem || q > kq) { k = l; kq = q; }
  }
  res[i] = k;
  keep[i] = kq >= mapq_threshold ? 1 : 0;
}

// ---- the text ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 sam_read_len(const OutSam &c, int mate) {  // what the CIGAR consumes of the read (I and M)
  u32 rl = 0;
  for (int q = 0; q < c.n_cigar[mate]; ++q) if ((c.cigar[mate][q] & 0xf) != 2) rl += c.cigar[mate][q] >> 4;
  return rl;
}
// base q of SEQ: the read as it is on +, PrepareNegativeSequenceAt of its first rl bases on - (sequence_batch.h:123-151)
__device__ __forceinline__ char sam_seq_at(const char *rseq, u32 rl, bool plus, u32 q) {
  if (plus) return rseq[q];
  switch (rseq[rl - 1 - q]) {
    case 'A': case 'a': return 'T';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    case 'T': case 't': return 'A';
    default: return 'N';
  }
}
// GenerateNMAndMDTag (alignment.cc:85-139) over the line's CIGAR: returns NM; *md_len = the MD string's length, written to md
// unless it is nullptr.  g = the reference from the line's position; reference bytes are printed as stored.
__device__ __forceinline__ u32 sam_nm_md(const OutSam &c, int mate, const u8 *g, const char *rseq, u32 rl, bool plus, char *md, u32 *md_len) {
  u32 nm = 0, nmatch = 0, rpos = 0, gpos = 0, ml = 0;
  auto number = [&](u32 v) { if (md) put_dec(md + ml, v); ml += dec_digits(v); };
  for (int q = 0; q < c.n_cigar[mate]; ++q) {
    const u32 op = c.cigar[mate][q] & 0xf, ol = c.cigar[mate][q] >> 4;
    if (op == 0) {
      for (u32 t = 0; t < ol; ++t, ++rpos, ++gpos) {
        const int gb = (signed char)g[gpos], sb = (signed char)sam_seq_at(rseq, rl, plus, rpos);
        if (gb == sb || gb - 'a' + 'A' == sb) ++nmatch;
        else { ++nm; number(nmatch); nmatch = 0; if (md) md[ml] = (char)gb; ++ml; }
      }
    } else if (op == 1) { nm += ol; rpos += ol; }
    else {
      nm += ol; number(nmatch); nmatch = 0;
      if (md) md[ml] = '^';
      ++ml;
      for (u32 t = 0; t < ol; ++t, ++ml) if (md) md[ml] = (char)g[gpos + t];
      gpos += ol;
    }
  }
  number(nmatch);
  *md_len = ml;
  return nm;
}
__device__ __forceinline__ int sam_int_digits(int v) { return v < 0 ? 1 + dec_digits((u32)(-(long long)v)) : dec_digits((u32)v); }
__device__ __forceinline__ char *sam_put_int(char *p, int v) {
  if (v < 0) { *p++ = '-'; return put_dec(p, (u32)(-(long long)v)); }
  return put_dec(p, (u32)v);
}
// "FLAG\tRNAME\tPOS\tMAPQ\tCIGAR\tRNEXT\tPNEXT\tTLEN\t" (the fields between the read name's tab and SEQ): written to p unless
// it is nullptr; returns its length
__device__ __forceinline__ u32 sam_mid_fields(const SamText &T, const SamLine &s, const OutSam &c, char *p) {
  char *const p0 = p;
  u32 l = 0;
  auto name = [&](u32 rid) {
    const u32 a = T.ref_name_off[rid], b = T.ref_name_off[rid + 1];
    if (p0) for (u32 k = a; k < b; ++k) p[l + k - a] = T.ref_names[k];
    l += b - a;
  };
  auto dec = [&](u32 v) { if (p0) put_dec(p + l, v); l += dec_digits(v); };
  auto ch = [&](char x) { if (p0) p[l] = x; ++l; };
  dec((u32)s.flag); ch('\t');
  name(s.rid); ch('\t');
  dec(s.pos + 1u); ch('\t');
  dec((u32)s.mapq); ch('\t');
  if (c.n_cigar[s.mate] == 0) ch('*');
  for (int q = 0; q < c.n_cigar[s.mate]; ++q) { dec(c.cigar[s.mate][q] >> 4); ch("MIDNSHP=XB"[c.cigar[s.mate][q] & 0xf]); }
  ch('\t');
  if (s.mrid < 0) ch('*');
  else if ((u32)s.mrid == s.rid) ch('=');
  else name((u32)s.mrid);
  ch('\t');
  dec(s.mrid < 0 ? 0u : s.mpos + 1u); ch('\t');
  if (p0) sam_put_int(p + l, s.tlen);
  l += sam_int_digits(s.tlen);
  ch('\t');
  return l;
}
struct SamLineView {  // what both passes derive from a line id
  SamLine s;
  const OutSam *c;
  const SamReads *R;
  const char *rseq;
  u64 full;
  u32 ri, rl;
  bool plus;
};
__device__ __forceinline__ SamLineView sam_view(const SamText &T, u32 l) {
  SamLineView v;
  v.s = sam_line(T, l);
  v.c = &T.cores[v.s.core];
  v.R = &T.r[v.s.mate];
  v.ri = v.s.read_id - T.first_read_id;
  v.rseq = v.R->seq + v.R->off[v.ri];
  v.full = v.R->off[v.ri + 1] - v.R->off[v.ri];
  v.rl = sam_read_len(*v.c, v.s.mate);
  v.plus = v.c->strand[v.s.mate] != 0;
  return v;
}
// Length pass, one thread per output line: len[i], nm[i]; err[1] counts CIGARs longer than their read; the translation's
// missing segments counted as bed_len_kernel does.
__global__ void sam_len_kernel(SamText T, const u32 *sel, u64 m, u32 *len, u32 *nm, int *err, BedTranslation Tr) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const SamLineView v = sam_view(T, sel[i]);
  if (v.rl > v.full) { atomicAdd(err + 1, 1); len[i] = 0; nm[i] = 0; return; }
  u32 md_len;
  const u32 x = sam_nm_md(*v.c, v.s.mate, T.ref + T.ref_off[v.s.rid] + v.s.pos, v.rseq, v.rl, v.plus, nullptr, &md_len);
  u32 l = (u32)(v.R->name_off[v.ri + 1] - v.R->name_off[v.ri]) + 1 + sam_mid_fields(T, v.s, *v.c, nullptr) + v.rl + 1 + (v.R->qual ? v.rl : 0) +
          6 + dec_digits(x) + 6 + md_len + 1;
  if (T.bcs) {
    u32 n_missing = 0;
    l += 6 + bed_barcode_field(Tr, T.bcs[v.s.core], T.bc_len, nullptr, &n_missing);
    if (n_missing) { atomicAdd(Tr.n_missing, (unsigned long long)n_missing); atomicMin(Tr.first_missing, (unsigned)i); }
  }
  len[i] = l;
  nm[i] = x;
}
// Write pass, one warp per line: the lanes copy the read name, SEQ and QUAL; lane 0 writes the other fields.  Every lane works
// out the positions itself, so the lanes never wait for each other.  off = the scan of len over the call, base = off of the
// chunk's first line (its byte 0 in out).
__global__ void sam_write_kernel(SamText T, const u32 *sel, u64 m, const u64 *off, u64 base, const u32 *nm, char *out, BedTranslation Tr) {
  const u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const u32 lane = threadIdx.x & 31u;
  if (i >= m) return;
  const SamLineView v = sam_view(T, sel[i]);
  char *p = out + (off[i] - base);
  const u64 na = v.R->name_off[v.ri], nb = v.R->name_off[v.ri + 1];
  for (u64 k = lane; k < nb - na; k += 32) p[k] = v.R->names[na + k];
  p += nb - na;
  const u32 mid = sam_mid_fields(T, v.s, *v.c, nullptr);
  if (lane == 0) { *p = '\t'; sam_mid_fields(T, v.s, *v.c, p + 1); }
  p += 1 + mid;
  for (u32 k = lane; k < v.rl; k += 32) p[k] = sam_seq_at(v.rseq, v.rl, v.plus, k);
  p += v.rl;
  if (lane == 0) *p = '\t';
  ++p;
  if (v.R->qual) {  // SAMMapping's constructor: the whole quality string reversed on -, then cut to SEQ's length
    const char *q = v.R->qual + v.R->off[v.ri];
    for (u32 k = lane; k < v.rl; k += 32) p[k] = v.plus ? q[k] : q[v.full - 1 - k];
    p += v.rl;
  }
  if (lane) return;
  const u32 x = nm[i];
  *p++ = '\t'; *p++ = 'N'; *p++ = 'M'; *p++ = ':'; *p++ = 'i'; *p++ = ':';
  p = put_dec(p, x);
  *p++ = '\t'; *p++ = 'M'; *p++ = 'D'; *p++ = ':'; *p++ = 'Z'; *p++ = ':';
  u32 md_len;
  sam_nm_md(*v.c, v.s.mate, T.ref + T.ref_off[v.s.rid] + v.s.pos, v.rseq, v.rl, v.plus, p, &md_len);
  p += md_len;
  if (T.bcs) {
    *p++ = '\t'; *p++ = 'C'; *p++ = 'B'; *p++ = ':'; *p++ = 'Z'; *p++ = ':';
    u32 n_missing = 0;  // none: the length pass found every segment
    p += bed_barcode_field(Tr, T.bcs[v.s.core], T.bc_len, p, &n_missing);
  }
  *p = '\n';
}
