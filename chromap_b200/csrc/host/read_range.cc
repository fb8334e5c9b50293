// chromap_b200 host side — --read-format: the parser (chromap.cc:825-865, sequence_effective_range.h:20-76) with the
// grammar made strict, and the in-place cut of one read (sequence_effective_range.h:80-118) for the host reader and the
// barcode pre-pass.  The device does the same cut while it packs FASTQ records (ingest.cuh).
#include <cstdint>
#include <cstring>

#include "read_range.h"

bool cmxhost::ReadRangeRepresentable(const cmx_read_range &r) {
  if (r.n < 1 || r.n > CMX_MAX_READ_RANGES) return false;
  for (uint32_t k = 0; k < r.n; ++k) {
    if (r.start[k] < 0 || (r.end[k] < r.start[k] && !(r.end[k] == -1 && k + 1 == r.n))) return false;
    if (k > 0 && r.start[k] <= r.end[k - 1]) return false;  // ascending, disjoint (end[k - 1] != -1 here)
  }
  return true;
}

namespace {

// a decimal field: digits only (start), or digits / "-1" (end); at most 9 digits so that it fits the reference's int
bool Number(const char *s, size_t n, bool allow_minus_one, int32_t *v) {
  if (allow_minus_one && n == 2 && s[0] == '-' && s[1] == '1') { *v = -1; return true; }
  if (n == 0 || n > 9) return false;
  int32_t x = 0;
  for (size_t i = 0; i < n; ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    x = x * 10 + (s[i] - '0');
  }
  *v = x;
  return true;
}

// one field "r1|r2|bc:start:end[:strand]" of length n
bool ParseField(const char *s, size_t n, cmx_read_range *r[3], bool named[3], bool *too_many) {
  if (n < 3 || s[2] != ':') return false;
  const int which = !strncmp(s, "r1", 2) ? 0 : !strncmp(s, "r2", 2) ? 1 : !strncmp(s, "bc", 2) ? 2 : -1;
  if (which < 0) return false;
  const char *part[3];
  size_t len[3], np = 0;
  for (size_t i = 3, b = 3; i <= n; ++i)
    if (i == n || s[i] == ':') {
      if (np == 3) return false;
      part[np] = s + b; len[np] = i - b; ++np;
      b = i + 1;
    }
  if (np < 2) return false;
  int32_t start, end;
  if (!Number(part[0], len[0], false, &start) || !Number(part[1], len[1], true, &end) || (end != -1 && end < start)) return false;
  if (np == 3 && (len[2] != 1 || (part[2][0] != '+' && part[2][0] != '-'))) return false;
  cmx_read_range &x = *r[which];
  if (!named[which]) { x.n = 0; named[which] = true; }
  if (np == 3) x.reverse = part[2][0] == '-';
  if (x.n == CMX_MAX_READ_RANGES) *too_many = true;
  else { x.start[x.n] = start; x.end[x.n] = end; ++x.n; }
  return true;
}

// utils.h:87-100: CharToUint8, complement, Uint8ToChar
char Complement(char c) {
  switch (c) {
    case 'A': case 'a': return 'T';
    case 'C': case 'c': return 'G';
    case 'G': case 'g': return 'C';
    case 'T': case 't': return 'A';
    default: return 'N';
  }
}

void Reverse(char *s, uint32_t n) {
  for (uint32_t i = 0, j = n; i + 1 < j; ++i, --j) { const char t = s[i]; s[i] = s[j - 1]; s[j - 1] = t; }
}

}  // namespace

extern "C" int cmx_parse_read_format(const char *fmt, cmx_read_range *r1, cmx_read_range *r2, cmx_read_range *bc) {
  if (!fmt || !r1 || !r2 || !bc) return CMX_ERR_INVALID;
  cmx_read_range *r[3] = {r1, r2, bc};
  bool named[3] = {false, false, false}, too_many = false;
  for (cmx_read_range *x : r) { memset(x, 0, sizeof(*x)); x->n = 1; x->end[0] = -1; }
  const size_t n = strlen(fmt);
  for (size_t i = 0; i < n;) {  // an empty string is no format at all (chromap.cc:826-828)
    size_t j = i;
    while (j < n && fmt[j] != ',') ++j;
    if (!ParseField(fmt + i, j - i, r, named, &too_many)) return CMX_ERR_INVALID;
    if (j == n) break;
    i = j + 1;
    if (i == n) return CMX_ERR_INVALID;  // a trailing comma
  }
  if (too_many) return CMX_ERR_READ_RANGE;
  for (cmx_read_range *x : r)
    if (!cmxhost::ReadRangeRepresentable(*x)) return CMX_ERR_READ_RANGE;
  return CMX_OK;
}

extern "C" int64_t cmx_apply_read_range(const cmx_read_range *range, char *seq, char *qual, uint32_t len) {
  if (!range || !cmxhost::ReadRangeRepresentable(*range) || (!seq && len)) return CMX_ERR_INVALID;
  const cmx_read_range &r = *range;
  for (uint32_t k = 0; k < r.n; ++k)
    if (r.end[k] != -1 && (uint32_t)r.end[k] >= len) return CMX_ERR_READ_RANGE;
  uint32_t m = 0;  // Replace: ranges copied forward in place (they ascend, so no byte is read after it was overwritten)
  for (uint32_t k = 0; k < r.n; ++k) {
    const uint32_t a = (uint32_t)r.start[k], e = r.end[k] == -1 ? len : (uint32_t)r.end[k] + 1;
    for (uint32_t j = a; j < e; ++j, ++m) {
      seq[m] = seq[j];
      if (qual) qual[m] = qual[j];
    }
  }
  if (r.reverse) {
    for (uint32_t i = 0; i < m; ++i) seq[i] = Complement(seq[i]);
    Reverse(seq, m);
    if (qual) Reverse(qual, m);
  }
  return m;
}
