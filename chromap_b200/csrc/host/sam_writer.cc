// chromap_b200 host side — SAM text from the device's SAM cores (cmx_sam_record): flags, mate fields and TLEN
// (mapping_generator.h:613-640, mapping_generator.cc:84-107), NM / MD (alignment.cc:85-139), record order, duplicate
// removal and MAPQ filter (sam_mapping.h:188-199, mapping_processor.h:161-202, mapping_writer.h:166-376, :405-437) and the
// lines themselves (mapping_writer.cc:312-356), with the cell barcode for barcoded runs.  No device needed; the device writes the
// same text in sam_text.cuh, and this writer stays the specification it is tested against.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../../include/chromap_b200.h"

namespace {
struct Line {
  const cmx_sam_record *core;
  int mate;  // 0 / 1: which span of the core
  int64_t pos, mpos;
  int rid, mrid, flag, tlen, mapq;
  uint32_t read_id;
  uint64_t bc;  // cell barcode key (0: bulk)
};
inline int BaseCode(char c) {  // utils.h:87-104
  switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; }
}
}  // namespace

// One writer for bulk and barcoded cores.  barcode_keys (NULL: bulk) is one key per core: it joins the order and the duplicate
// test (sam_mapping.h:188-199) and is written as CB:Z: (mapping_writer.cc:350-354) through `tr` (NULL: the key's bases).
static int64_t FormatSam(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const char *ref_concat,
                         const uint64_t *ref_offsets, const cmx_sam_record *records, const uint64_t *barcode_keys, uint32_t bc_len, uint64_t n,
                         const cmx_read_set *reads1, const cmx_read_set *reads2, uint32_t first_read_id, const cmx_barcode_translation *tr, char *buf,
                         int64_t cap) {
  if (!p || !ref_names || !ref_lengths || !ref_concat || !ref_offsets || (!records && n) || !reads1) return -1;
  if (barcode_keys && (bc_len == 0 || bc_len > 32)) return -1;
  if (barcode_keys && tr && (tr->from_len < 1 || tr->from_len > 31 || (tr->n && (!tr->keys || !tr->to_off)))) return -1;
  const bool pe = reads2 != nullptr;
  std::vector<Line> lines;
  lines.reserve(n * (pe ? 2 : 1));
  for (uint64_t i = 0; i < n; ++i) {
    const cmx_sam_record &c = records[i];
    if (c.overflow) return -2;
    const uint64_t bc = barcode_keys ? barcode_keys[i] : 0;
    if (!pe) {
      lines.push_back({&c, 0, (int64_t)c.pos[0], 0, (int)c.rid, -1, (c.strand[0] ? 0 : 16) | (c.secondary ? 256 : 0), 0, (int)c.mapq, c.read_id, bc});
      continue;
    }
    int f1 = 3 | 64, f2 = 3 | 128;
    if (!c.strand[0]) { f1 |= 16; f2 |= 32; }
    if (!c.strand[1]) { f1 |= 32; f2 |= 16; }
    if (c.secondary) { f1 |= 256; f2 |= 256; }
    const int tlen = c.strand[0] ? (int)(c.end[1] - c.pos[0] + 1u) : (int)(c.end[0] - c.pos[1] + 1u);  // PairedEndMappingInMemory::GetFragmentLength
    lines.push_back({&c, 0, (int64_t)c.pos[0], (int64_t)c.pos[1], (int)c.rid, (int)c.rid, f1, c.strand[0] ? tlen : -tlen, (int)c.mapq, c.read_id, bc});
    lines.push_back({&c, 1, (int64_t)c.pos[1], (int64_t)c.pos[0], (int)c.rid, (int)c.rid, f2, c.strand[1] ? tlen : -tlen, (int)c.mapq, c.read_id, bc});
  }
  auto key = [](const Line &l) { return std::make_tuple(l.rid, l.pos, l.bc, l.mrid, l.mpos, l.flag & 64, l.mapq, l.read_id); };
  std::stable_sort(lines.begin(), lines.end(), [&](const Line &a, const Line &b) { return key(a) < key(b); });
  auto same = [](const Line &a, const Line &b) {
    return a.rid == b.rid && a.pos == b.pos && a.bc == b.bc && (a.flag & 64) == (b.flag & 64) && a.mrid == b.mrid && a.mpos == b.mpos;
  };
  std::vector<const Line *> keep;
  if (p->remove_pcr_duplicates) {
    size_t i = 0;
    while (i < lines.size()) {
      size_t j = i + 1, k = i;
      for (; j < lines.size() && same(lines[j], lines[j - 1]); ++j) {
        if (p->low_memory_mode) { if (lines[j].mapq > lines[k].mapq) k = j; } else k = j;
      }
      if (lines[k].mapq >= p->mapq_threshold) keep.push_back(&lines[k]);
      i = j;
    }
  } else for (const Line &l : lines) if (l.mapq >= p->mapq_threshold) keep.push_back(&l);
  auto read_of = [&](const Line &l, const char **rseq, size_t *full, uint32_t *ri) {
    const cmx_read_set &rs = l.mate == 0 ? *reads1 : *reads2;
    *ri = l.core->read_id - first_read_id;
    *rseq = rs.seq + rs.off[*ri];
    *full = (size_t)(rs.off[*ri + 1] - rs.off[*ri]);
    size_t rl = 0;  // the mapped read may be shorter than the record (adapter trimming keeps a prefix): its length is what the CIGAR consumes
    for (int q = 0; q < l.core->n_cigar[l.mate]; ++q) if ((l.core->cigar[l.mate][q] & 0xf) != 2) rl += l.core->cigar[l.mate][q] >> 4;
    return rl;
  };
  // the checks come before any text: a CIGAR longer than its read, then a barcode segment without a translation
  for (const Line *l : keep) {
    const char *rseq; size_t full; uint32_t ri;
    if (read_of(*l, &rseq, &full, &ri) > full) return -3;
  }
  std::unordered_map<uint64_t, uint64_t> at;
  if (barcode_keys && tr) for (uint64_t i = 0; i < tr->n; ++i) at[tr->keys[i]] = i;
  auto cell_barcode = [&](uint64_t bc, std::string *out) {  // BarcodeTranslator::Translate (barcode_translator.h:72-123)
    out->clear();
    if (!tr) { for (uint32_t j = 0; j < bc_len; ++j) out->push_back("ACGT"[(bc >> ((bc_len - 1 - j) * 2)) & 3]); return true; }
    const uint32_t L = tr->from_len, nseg = bc_len / L;
    const uint64_t mask = (1ull << (2 * L)) - 1;
    for (uint32_t s = 0; s < nseg; ++s) {
      auto it = at.find((bc >> (2 * L * (nseg - 1 - s))) & mask);
      if (it == at.end()) return false;
      if (s) out->push_back('-');
      out->append(tr->to + tr->to_off[it->second], tr->to_off[it->second + 1] - tr->to_off[it->second]);
    }
    return true;
  };
  std::string cb;
  if (barcode_keys && tr)
    for (const Line *l : keep) if (!cell_barcode(l->bc, &cb)) return CMX_ERR_BARCODE_TRANSLATE;
  int64_t len = 0;
  auto put = [&](const std::string &s) {
    if (buf && len + (int64_t)s.size() <= cap) memcpy(buf + len, s.data(), s.size());
    len += (int64_t)s.size();
  };
  for (uint32_t i = 0; i < n_seq; ++i) put(std::string("@SQ\tSN:") + ref_names[i] + "\tLN:" + std::to_string(ref_lengths[i]) + "\n");
  std::string seq, qual, cig, md, out;
  for (const Line *l : keep) {
    const cmx_sam_record &c = *l->core;
    const cmx_read_set &rs = l->mate == 0 ? *reads1 : *reads2;
    const char *rseq;
    size_t full;
    uint32_t ri;
    const size_t rl = read_of(*l, &rseq, &full, &ri);
    const bool plus = c.strand[l->mate] != 0;
    if (plus) seq.assign(rseq, rl);
    else {  // PrepareNegativeSequenceAt on the kept prefix (sequence_batch.h:123-151)
      seq.resize(rl);
      for (size_t q = 0; q < rl; ++q) { const int b = BaseCode(rseq[rl - 1 - q]); seq[q] = b < 4 ? "ACGT"[3 - b] : 'N'; }
    }
    qual.clear();
    if (rs.qual) {  // SAMMapping's constructor: reverse the whole quality string for the - strand, then cut to the sequence length
      qual.assign(rs.qual + rs.off[ri], full);
      if (!plus) std::reverse(qual.begin(), qual.end());
      qual.resize(rl);
    }
    cig.clear(); md.clear();
    int nm = 0, nmatch = 0;
    size_t rpos = 0, gpos = 0;
    const char *g = ref_concat + ref_offsets[c.rid] + c.pos[l->mate];
    for (int q = 0; q < c.n_cigar[l->mate]; ++q) {  // GenerateNMAndMDTag
      const uint32_t op = c.cigar[l->mate][q] & 0xf, ol = c.cigar[l->mate][q] >> 4;
      cig += std::to_string(ol); cig.push_back("MIDNSHP=XB"[op]);
      if (op == 0) {
        for (uint32_t t = 0; t < ol; ++t, ++rpos, ++gpos) {
          if (g[gpos] == seq[rpos] || g[gpos] - 'a' + 'A' == seq[rpos]) ++nmatch;
          else { ++nm; md += std::to_string(nmatch); nmatch = 0; md.push_back(g[gpos]); }
        }
      } else if (op == 1) { nm += (int)ol; rpos += ol; }
      else { nm += (int)ol; md += std::to_string(nmatch); nmatch = 0; md.push_back('^'); for (uint32_t t = 0; t < ol; ++t) md.push_back(g[gpos++]); }
    }
    md += std::to_string(nmatch);
    if (cig.empty()) cig = "*";
    out.assign(rs.names[ri]);
    out += "\t" + std::to_string(l->flag) + "\t" + ref_names[l->rid] + "\t" + std::to_string(l->pos + 1) + "\t" + std::to_string(l->mapq) + "\t" + cig + "\t";
    out += l->mrid < 0 ? "*" : (l->mrid == l->rid ? "=" : ref_names[l->mrid]);
    out += "\t" + std::to_string(l->mrid < 0 ? 0 : l->mpos + 1) + "\t" + std::to_string(l->tlen) + "\t" + seq + "\t" + qual + "\tNM:i:" + std::to_string(nm) + "\tMD:Z:" + md;
    if (barcode_keys) { cell_barcode(l->bc, &cb); out += "\tCB:Z:" + cb; }
    out += "\n";
    put(out);
  }
  return len;
}

extern "C" int64_t cmx_format_sam(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const char *ref_concat,
                                  const uint64_t *ref_offsets, const cmx_sam_record *records, uint64_t n, const cmx_read_set *reads1,
                                  const cmx_read_set *reads2, uint32_t first_read_id, char *buf, int64_t cap) {
  return FormatSam(p, ref_names, ref_lengths, n_seq, ref_concat, ref_offsets, records, nullptr, 0, n, reads1, reads2, first_read_id, nullptr, buf, cap);
}

extern "C" int64_t cmx_format_sam_bc(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const char *ref_concat,
                                     const uint64_t *ref_offsets, const cmx_sam_record *records, const uint64_t *barcode_keys, uint32_t bc_len, uint64_t n,
                                     const cmx_read_set *reads1, const cmx_read_set *reads2, uint32_t first_read_id,
                                     const cmx_barcode_translation *translation, char *buf, int64_t cap) {
  return FormatSam(p, ref_names, ref_lengths, n_seq, ref_concat, ref_offsets, records, barcode_keys, bc_len, n, reads1, reads2, first_read_id, translation, buf,
                   cap);
}

// PAF text (mapping_writer.cc:177-196 single-end, :249-310 paired-end) from the BED-path records: PAFMapping /
// PairedPAFMapping carry the same fields plus read names and (trimmed) read lengths.  Order, duplicate rule, Tn5 shift and
// MAPQ filter are the PAF types' own (paf_mapping.h) -- including what EmplaceBackPairedEndMappingRecord<PairedPAFMapping>
// (mapping_generator.cc:146-167) does to the fields: it passes (start, negative alignment length, fragment length,
// positive alignment length) to a constructor that takes (start, fragment length, positive, negative), and both mates'
// MAPQs were overwritten with the pair's (mapping_generator.h:611-612).  No device needed.
extern "C" int64_t cmx_format_paf(const cmx_params *p, const char *const *ref_names, const uint32_t *ref_lengths, const cmx_pe_record *records, uint64_t n,
                                  const char *const *names1, const uint16_t *lengths1, const char *const *names2, const uint16_t *lengths2,
                                  uint32_t first_read_id, char *buf, int64_t cap) {
  if (!p || !ref_names || !ref_lengths || (!records && n) || !names1 || !lengths1) return -1;
  const bool se = names2 == nullptr;
  if (!se && !lengths2) return -1;
  struct Rec { uint32_t read_id, rid, start; uint16_t frag, pal, nal; uint8_t mapq, dir, uniq, dups; };
  std::vector<Rec> recs(n);
  for (uint64_t i = 0; i < n; ++i) {
    const cmx_pe_record &r = records[i];
    Rec &o = recs[i];
    o.read_id = r.read_id; o.rid = r.rid; o.start = r.fragment_start; o.mapq = r.mapq; o.dir = r.direction; o.uniq = r.is_unique; o.dups = r.num_dups;
    if (se) { o.frag = r.fragment_length; o.pal = o.nal = 0; }
    else { o.frag = r.negative_alignment_length; o.pal = r.fragment_length; o.nal = r.positive_alignment_length; }
  }
  auto tn5 = [&](Rec &r) {
    if (se) { if (r.dir == 1) r.start += 4; else r.frag -= 5; }
    else { r.start += 4; r.pal -= 4; r.frag -= 9; r.nal -= 5; }
  };
  if (!p->low_memory_mode && p->tn5_shift) for (auto &r : recs) tn5(r);
  auto key = [&](const Rec &r) {  // PAFMapping: (start, length, mapq, direction, unique, read id, read length); paired: mapq1 = mapq2 = mapq
    return std::make_tuple(r.rid, r.start, r.frag, r.mapq, r.dir, r.uniq, r.read_id, r.pal, r.nal);
  };
  std::stable_sort(recs.begin(), recs.end(), [&](const Rec &a, const Rec &b) { return key(a) < key(b); });
  auto same = [&](const Rec &a, const Rec &b) { return a.rid == b.rid && a.start == b.start && (se || a.frag == b.frag); };
  int64_t len = 0;
  char line[4096];
  size_t i = 0;
  while (i < recs.size()) {
    size_t j = i + 1, k = i;
    uint32_t dups = 1;
    if (p->remove_pcr_duplicates)
      for (; j < recs.size() && same(recs[j], recs[j - 1]); ++j) {
        ++dups;
        if (p->low_memory_mode) { if (recs[j].mapq > recs[k].mapq) k = j; } else k = j;
      }
    Rec r = recs[k];
    i = j;
    if (r.mapq < p->mapq_threshold) continue;
    if (p->low_memory_mode && p->tn5_shift) tn5(r);
    const uint32_t ri = r.read_id - first_read_id;
    const char *rn = ref_names[r.rid];
    const uint32_t rl = ref_lengths[r.rid];
    int l;
    if (se) {
      l = snprintf(line, sizeof(line), "%s\t%u\t0\t%u\t%c\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", names1[ri], (uint32_t)lengths1[ri], (uint32_t)lengths1[ri], r.dir ? '+' : '-', rn,
                   rl, r.start, (uint32_t)(r.start + r.frag), (uint32_t)lengths1[ri], (uint32_t)r.frag, (uint32_t)r.mapq);
    } else {
      const uint32_t pos_end = r.start + r.pal, neg_end = r.start + r.frag, neg_start = neg_end - r.nal;
      const uint32_t l1 = lengths1[ri], l2 = lengths2[ri];
      if (r.dir)
        l = snprintf(line, sizeof(line), "%s\t%u\t0\t%u\t+\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n%s\t%u\t0\t%u\t-\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", names1[ri], l1, l1, rn, rl, r.start,
                     pos_end, l1, (uint32_t)r.pal, (uint32_t)r.mapq, names2[ri], l2, l2, rn, rl, neg_start, neg_end, l2, (uint32_t)r.nal, (uint32_t)r.mapq);
      else
        l = snprintf(line, sizeof(line), "%s\t%u\t0\t%u\t-\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n%s\t%u\t0\t%u\t+\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", names1[ri], l1, l1, rn, rl, neg_start,
                     neg_end, l1, (uint32_t)r.nal, (uint32_t)r.mapq, names2[ri], l2, l2, rn, rl, r.start, pos_end, l2, (uint32_t)r.pal, (uint32_t)r.mapq);
    }
    if (l < 0 || l >= (int)sizeof(line)) return -2;
    if (buf && len + l <= cap) memcpy(buf + len, line, l);
    len += l;
    (void)dups;
  }
  return len;
}
