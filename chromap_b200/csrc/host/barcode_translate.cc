// chromap_b200 host side — --barcode-translate: the table parser (BarcodeTranslator::SetTranslateTable and
// ProcessTranslateFileLine, barcode_translator.h:42-68,125-145) made strict, and the translated barcoded BED text
// (mapping_writer.cc:18-24,131-137 through Translate, barcode_translator.h:72-101) for hosts without the device writer.
// The device writes the same text in bed_len_kernel / bed_write_kernel (postprocess.cuh).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/chromap_b200.h"

namespace {

int Refuse(char *err, uint64_t err_cap, uint64_t line, const char *why) {
  if (err && err_cap) snprintf(err, err_cap, "line %llu: %s", (unsigned long long)line, why);
  return CMX_ERR_INVALID;
}

// utils.h:87-93 for the bytes the parser lets through
int BaseCode(char c) {
  switch (c) {
    case 'A': case 'a': return 0;
    case 'C': case 'c': return 1;
    case 'G': case 'g': return 2;
    case 'T': case 't': return 3;
    default: return -1;
  }
}

}  // namespace

extern "C" int cmx_parse_barcode_translation(const char *text, uint64_t n_bytes, cmx_barcode_translation *out, char *err, uint64_t err_cap) {
  if (!out || (!text && n_bytes)) return CMX_ERR_INVALID;
  memset(out, 0, sizeof(*out));
  if (n_bytes == 0) return Refuse(err, err_cap, 0, "the table has no lines");
  std::vector<uint64_t> keys;
  std::vector<std::string> to;
  std::unordered_map<uint64_t, size_t> at;
  int64_t from_len = -1;
  uint64_t line = 0;
  for (uint64_t b = 0; b < n_bytes;) {
    uint64_t e = b;
    while (e < n_bytes && text[e] != '\n') ++e;
    ++line;
    const char *s = text + b;
    const uint64_t len = e - b;
    b = e + 1;  // past the newline (or the end)
    if (len > 510) return Refuse(err, err_cap, line, "longer than 510 bytes (the reference reads it in 512-byte pieces)");
    if (memchr(s, 0, len)) return Refuse(err, err_cap, line, "a NUL byte");
    if (len == 0) return Refuse(err, err_cap, line, "an empty line");
    uint64_t sep = 0;
    while (sep < len && s[sep] != ',' && s[sep] != '\t') ++sep;
    if (sep == len) return Refuse(err, err_cap, line, "no ',' or tab between TO and FROM");
    const uint64_t fl = len - sep - 1;
    if (fl == 0) return Refuse(err, err_cap, line, "an empty FROM barcode");
    if (fl >= 32) return Refuse(err, err_cap, line, "a FROM barcode of 32 bases or more");
    if (from_len >= 0 && (int64_t)fl != from_len) return Refuse(err, err_cap, line, "a FROM barcode whose length differs from the lines before it");
    from_len = (int64_t)fl;
    uint64_t key = 0;
    for (uint64_t i = sep + 1; i < len; ++i) {
      const int c = BaseCode(s[i]);
      if (c < 0) return Refuse(err, err_cap, line, "a FROM byte other than A, C, G, T (either case)");
      key = (key << 2) | (uint64_t)c;
    }
    auto it = at.find(key);
    if (it == at.end()) { at.emplace(key, keys.size()); keys.push_back(key); to.emplace_back(s, sep); }
    else to[it->second].assign(s, sep);  // kh_put on an existing key: the later line wins
  }
  const uint64_t n = keys.size();
  uint64_t total = 0;
  for (const auto &t : to) total += t.size();
  out->keys = (uint64_t *)malloc(n * sizeof(uint64_t));
  out->to_off = (uint64_t *)malloc((n + 1) * sizeof(uint64_t));
  out->to = (char *)malloc(total + 1);
  if (!out->keys || !out->to_off || !out->to) { cmx_free_barcode_translation(out); return Refuse(err, err_cap, 0, "out of memory"); }
  out->to_off[0] = 0;
  for (uint64_t i = 0; i < n; ++i) {
    out->keys[i] = keys[i];
    memcpy(out->to + out->to_off[i], to[i].data(), to[i].size());
    out->to_off[i + 1] = out->to_off[i] + to[i].size();
  }
  out->n = n;
  out->from_len = (uint32_t)from_len;
  return CMX_OK;
}

extern "C" void cmx_free_barcode_translation(cmx_barcode_translation *t) {
  if (!t) return;
  free(t->keys); free(t->to_off); free(t->to);
  memset(t, 0, sizeof(*t));
}

extern "C" int64_t cmx_format_bed_bc_tr(const char *const *names, const cmx_pe_record *recs, const uint64_t *bcs, uint64_t n, uint32_t bc_len,
                                        const cmx_barcode_translation *tr, char *buf, int64_t cap) {
  if (!names || (n && (!recs || !bcs)) || bc_len == 0 || bc_len > 32) return CMX_ERR_INVALID;
  if (!tr) return cmx_format_bed_bc(names, recs, bcs, n, bc_len, buf, cap);
  if (tr->from_len < 1 || tr->from_len > 31 || (tr->n && (!tr->keys || !tr->to_off))) return CMX_ERR_INVALID;
  std::unordered_map<uint64_t, uint64_t> at;
  for (uint64_t i = 0; i < tr->n; ++i) at[tr->keys[i]] = i;
  const uint32_t L = tr->from_len, nseg = bc_len / L;
  const uint64_t mask = (1ull << (2 * L)) - 1;
  std::vector<std::string> fields(n);
  for (uint64_t i = 0; i < n; ++i)
    for (uint32_t s = 0; s < nseg; ++s) {  // Translate's segment s: ((bc << 2sL) >> 2(nseg - 1)L) & mask
      auto it = at.find((bcs[i] >> (2 * L * (nseg - 1 - s))) & mask);
      if (it == at.end()) return CMX_ERR_BARCODE_TRANSLATE;
      if (s) fields[i] += '-';
      fields[i].append(tr->to + tr->to_off[it->second], tr->to_off[it->second + 1] - tr->to_off[it->second]);
    }
  int64_t len = 0;
  for (uint64_t i = 0; i < n; ++i) {  // mapping_writer.cc:131-137
    const cmx_pe_record &r = recs[i];
    const std::string line = std::string(names[r.rid]) + "\t" + std::to_string(r.fragment_start) + "\t" + std::to_string((uint32_t)(r.fragment_start + r.fragment_length)) +
                             "\t" + fields[i] + "\t" + std::to_string((uint32_t)r.num_dups) + "\n";
    if (buf && len + (int64_t)line.size() <= cap) memcpy(buf + len, line.data(), line.size());
    len += (int64_t)line.size();
  }
  return len;
}
