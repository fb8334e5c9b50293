// TEST INFRASTRUCTURE ONLY — see oracle_chromap.h.  CPU restatement of Chromap's paired-end
// mapping hot path in our own flat data layout.  File:line citations are into /root/reference/src.
#include "oracle_chromap.h"

#include <omp.h>
#include <zlib.h>

#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <random>
#include <string>
#include <tuple>
#include <vector>

typedef uint64_t u64;
typedef uint32_t u32;

// ----------------------------------------------------------------------------------------------
// Base coding (utils.h:87-104): A/a=0 C/c=1 G/g=2 T/t=3, everything else 4.
static uint8_t g_code[256];
static struct CodeInit {
  CodeInit() {
    memset(g_code, 4, sizeof(g_code));
    g_code['A'] = g_code['a'] = 0;
    g_code['C'] = g_code['c'] = 1;
    g_code['G'] = g_code['g'] = 2;
    g_code['T'] = g_code['t'] = 3;
  }
} g_code_init;
static inline uint8_t code(char c) { return g_code[(uint8_t)c]; }

// Invertible 64-bit mix (utils.h:76-85).
static inline u64 mix64(u64 key, u64 mask) {
  key = (~key + (key << 21)) & mask;
  key = key ^ key >> 24;
  key = ((key + (key << 3)) + (key << 8)) & mask;
  key = key ^ key >> 14;
  key = ((key + (key << 2)) + (key << 4)) & mask;
  key = key ^ key >> 28;
  key = (key + (key << 31)) & mask;
  return key;
}

struct Mm {
  u64 hash;
  u64 hit;  // ((seq_index<<32 | end_pos) << 1) | strand
};

// minimizer_generator.cc:7-139.  (k,w)-minimizers, strand-canonical, double-hashed key, N-aware.
static void gen_minimizers(const char *seq, u32 len, u32 seq_index, int k, int w, std::vector<Mm> &out) {
  const u64 shift = 2 * (k - 1);
  const u64 mask = (((u64)1) << (2 * k)) - 1;
  u64 fwd = 0, rev = 0;
  Mm ring[256];
  for (int i = 0; i < w; ++i) ring[i] = {UINT64_MAX, UINT64_MAX};
  Mm best = {UINT64_MAX, UINT64_MAX};
  int run = 0;       // unambiguous_length
  int slot = 0;      // position_in_buffer
  int best_slot = 0; // min_position
  for (u32 pos = 0; pos < len; ++pos) {
    const uint8_t b = code(seq[pos]);
    Mm cur = {UINT64_MAX, UINT64_MAX};
    if (b < 4) {
      fwd = ((fwd << 2) | b) & mask;
      rev = (rev >> 2) | (((u64)(3 ^ b)) << shift);
      if (fwd == rev) continue;  // :42-45 — skips ring write and ring advance too
      const u64 hf = mix64(fwd, mask), hr = mix64(rev, mask);
      const u64 strand = hf < hr ? 0 : 1;  // tie -> reverse (:51-52)
      ++run;
      if (run >= k) {
        cur.hash = mix64(strand ? hr : hf, mask);  // Hash64(Hash64(kmer)) (:55)
        cur.hit = ((((u64)seq_index) << 32 | pos) << 1) | strand;
      }
    } else {
      run = 0;
    }
    ring[slot] = cur;
    if (run == w + k - 1 && best.hash != UINT64_MAX && best.hash < cur.hash) {
      // first full window: identical k-mers not stored yet (:66-77)
      for (int j = slot + 1; j < w; ++j)
        if (best.hash == ring[j].hash && ring[j].hit != best.hit) out.push_back(ring[j]);
      for (int j = 0; j < slot; ++j)
        if (best.hash == ring[j].hash && ring[j].hit != best.hit) out.push_back(ring[j]);
    }
    if (cur.hash <= best.hash) {
      if (run >= w + k && best.hash != UINT64_MAX) out.push_back(best);
      best = cur;
      best_slot = slot;
    } else if (slot == best_slot) {
      if (run >= w + k - 1 && best.hash != UINT64_MAX) out.push_back(best);
      best.hash = UINT64_MAX;
      for (int j = slot + 1; j < w; ++j)
        if (best.hash >= ring[j].hash) { best = ring[j]; best_slot = j; }
      for (int j = 0; j <= slot; ++j)
        if (best.hash >= ring[j].hash) { best = ring[j]; best_slot = j; }
      if (run >= w + k - 1 && best.hash != UINT64_MAX) {
        for (int j = slot + 1; j < w; ++j)
          if (best.hash == ring[j].hash && best.hit != ring[j].hit) out.push_back(ring[j]);
        for (int j = 0; j <= slot; ++j)
          if (best.hash == ring[j].hash && best.hit != ring[j].hit) out.push_back(ring[j]);
      }
    }
    if (++slot == w) slot = 0;
  }
  if (best.hash != UINT64_MAX) out.push_back(best);
}

// ----------------------------------------------------------------------------------------------
struct orc_reference {
  std::vector<std::string> names;
  std::vector<std::string> seqs;  // each padded with 64 NULs past the end (kseq leaves a NUL + slack)
  std::vector<u32> lens;
};

struct orc_index {
  int k = 0, w = 0;
  u32 n_buckets = 0, size = 0, n_occupied = 0, upper_bound = 0;
  std::vector<u32> flags;
  std::vector<u64> keys, vals, occ;
  // khash.h:232-245 with hash = key>>1 truncated to 32 bit (index_utils.h:13-17), triangular probing.
  bool lookup(u64 mm_hash, u64 &key, u64 &val) const {
    if (!n_buckets) return false;
    const u64 q = mm_hash << 1;
    const u32 m = n_buckets - 1;
    u32 i = (u32)(q >> 1) & m, last = i, step = 0;
    for (;;) {
      const u32 f = (flags[i >> 4] >> ((i & 0xfU) << 1)) & 3;
      if (f & 2) return false;  // empty
      if (!(f & 1) && (keys[i] >> 1) == (q >> 1)) { key = keys[i]; val = vals[i]; return true; }
      i = (i + (++step)) & m;
      if (i == last) return false;
    }
  }
};

struct Cand {
  u64 pos;
  uint8_t cnt;
};
static inline bool cand_less(const Cand &a, const Cand &b) {  // candidate.h:23-33
  if (a.cnt != b.cnt) return a.cnt > b.cnt;
  return a.pos < b.pos;
}
struct Draft {
  int err;
  u64 pos;  // rid<<32 | end position
};

struct ReadState {  // mapping_metadata.h:24-175
  std::vector<Mm> mm;
  std::vector<u64> hits[2];     // [0]=positive [1]=negative
  std::vector<Cand> cand[2], buf[2];
  std::vector<Draft> map[2];
  std::vector<int> split[2];  // split_sites_, parallel to map[] (draft_mapping_generator.cc:550-554)
  int min_err, second_min_err, n_best, n_second_best;
  u32 rep_len;
  void reset() {
    mm.clear();
    for (int s = 0; s < 2; ++s) { hits[s].clear(); cand[s].clear(); buf[s].clear(); map[s].clear(); split[s].clear(); }
    rep_len = 0;
  }
};

struct RepStats {  // index_utils.h:21-26
  u32 len = 0, prev = UINT32_MAX;
  int count = 0;
};
static void rep_update(int k, int w, u32 read_pos, RepStats &st) {  // index.cc:507-523
  if (st.prev > read_pos) st.len += k;
  else if (read_pos < st.prev + k + w - 1) st.len += read_pos - st.prev;
  else st.len += k;
  st.prev = read_pos;
  ++st.count;
}
static inline u64 hit_to_candidate(int k, u64 ref_hit, u64 read_hit) {  // index.cc:491-505
  const u32 rp = (u32)(ref_hit >> 1), qp = (u32)(read_hit >> 1);
  const bool same = ((ref_hit ^ read_hit) & 1) == 0;
  const u32 start = same ? rp - qp : rp + qp - (u32)k + 1;  // u32 wrap kept
  return ((ref_hit >> 33) << 32) | start;
}

// index.cc:237-349.  Fills sorted +/- hit lists; returns repetitive seed count.
static int gen_hits(const orc_index &ix, u32 max_freq, u32 rep_freq, ReadState &rs) {
  RepStats st;
  for (const Mm &m : rs.mm) {
    u64 key, val;
    if (!ix.lookup(m.hash, key, val)) continue;
    if (key & 1) {
      rs.hits[((val ^ m.hit) & 1) ? 1 : 0].push_back(hit_to_candidate(ix.k, val, m.hit));
      continue;
    }
    const u32 n = (u32)val, off = (u32)(val >> 32);
    if (n < max_freq)
      for (u32 i = 0; i < n; ++i) {
        const u64 rh = ix.occ[off + i];
        rs.hits[((rh ^ m.hit) & 1) ? 1 : 0].push_back(hit_to_candidate(ix.k, rh, m.hit));
      }
    if (n >= rep_freq) rep_update(ix.k, ix.w, (u32)(m.hit >> 1), st);
  }
  // heap merge (round 2) and std::sort (round 1) yield the same sorted multiset (index.cc:317-333)
  std::sort(rs.hits[0].begin(), rs.hits[0].end());
  std::sort(rs.hits[1].begin(), rs.hits[1].end());
  rs.rep_len = st.len;
  return st.count;
}

// candidate_processor.cc:283-342.  Linear clustering scan; sentinel stays in `hits`.
static void cluster_hits(int e, int need, u32 n_mm, std::vector<u64> &hits, std::vector<Cand> &out) {
  hits.push_back(UINT64_MAX);
  int mcount = 1, eq = 1, best_eq = 1;
  u64 prev = hits[0], best = hits[0];
  u32 prev_rid = (u32)(prev >> 32), prev_pos = (u32)prev;
  for (size_t i = 1; i < hits.size(); ++i) {
    const u32 rid = (u32)(hits[i] >> 32), pos = (u32)hits[i];
    if (rid != prev_rid || pos > prev_pos + (u32)e ||
        ((u32)mcount >= n_mm && pos > (u32)best + (u32)e)) {
      if (mcount >= need) out.push_back({best, (uint8_t)best_eq});
      mcount = 1; eq = 1; best_eq = 1; best = hits[i];
    } else {
      if (hits[i] == best) { ++eq; ++best_eq; }
      else if (hits[i] == prev) { ++eq; if (eq > best_eq) { best = prev; best_eq = eq; } }
      else eq = 1;
      ++mcount;
    }
    prev = hits[i]; prev_rid = rid; prev_pos = pos;
  }
}

// candidate_processor.cc:12-71.
static void gen_candidates(const orc_params &P, const orc_index &ix, ReadState &rs) {
  rs.rep_len = 0;
  int rep = gen_hits(ix, P.max_seed_freq0, P.max_seed_freq0, rs);
  bool high = false;
  if (rs.hits[0].size() + rs.hits[1].size() == 0) {
    rs.hits[0].clear(); rs.hits[1].clear(); rs.rep_len = 0;
    rep = gen_hits(ix, P.max_seed_freq1, P.max_seed_freq0, rs);
    high = !(rs.hits[0].empty() || rs.hits[1].empty());
  }
  int need = (int)rs.mm.size() - rep;
  need = need > 1 ? need : 1;
  need = need > P.min_num_seeds ? P.min_num_seeds : need;
  if (high) need = P.min_num_seeds;
  cluster_hits(P.error_threshold, need, rs.mm.size(), rs.hits[0], rs.cand[0]);
  cluster_hits(P.error_threshold, need, rs.mm.size(), rs.hits[1], rs.cand[1]);
}

// index.cc:351-489: mate-guided lookup on one strand.  Returns +max count or -max count on bail-out.
// probe(i, key, val, hit): the table entry of minimizer i (false = absent) and its read-side hit word (position << 1 | strand);
// the mapper probes its khash index, the device tests hand in records that were probed elsewhere.
template <typename Probe>
static int rescue_core(int k, int w, int max_seed_freq0, int min_num_seeds, int strand, u32 range, size_t n_mm, Probe probe,
                       const u64 *occ, const std::vector<Cand> &mate, u32 &rep_len, std::vector<u64> &hits) {
  int max_cnt = 0, n_best = 0;
  for (const Cand &c : mate) {
    if (c.cnt > max_cnt) { max_cnt = c.cnt; n_best = 1; }
    else if (c.cnt == max_cnt) ++n_best;
  }
  if (n_best >= 300 || mate.size() > (size_t)max_seed_freq0 ||
      (max_cnt <= min_num_seeds && n_best >= 200))
    return -max_cnt;
  std::vector<std::pair<u64, u64>> win;
  for (const Cand &c : mate)
    if (c.cnt == max_cnt) win.push_back({c.pos < range ? 0 : c.pos - range, c.pos + range});
  if (win.empty()) return max_cnt;
  size_t nw = 1;
  for (size_t i = 1; i < win.size(); ++i) {
    if (win[nw - 1].second < win[i].first) win[nw++] = win[i];
    else win[nw - 1].second = win[i].second;
  }
  win.resize(nw);
  RepStats st;
  for (size_t mi = 0; mi < n_mm; ++mi) {
    u64 key, val, mhit;
    if (!probe(mi, key, val, mhit)) continue;
    if (key & 1) {
      const bool same = ((val ^ mhit) & 1) == 0;
      if ((same && strand == 0) || (!same && strand == 1)) hits.push_back(hit_to_candidate(k, val, mhit));
      continue;
    }
    const u32 off = (u32)(val >> 32), n = (u32)val;
    int32_t prev_l = 0;
    for (size_t bi = 0; bi < nw; ++bi) {
      int32_t l = prev_l, mid = 0, r = (int32_t)n - 1;
      const u64 lo = win[bi].first;
      while (l <= r) {  // index.cc:447-459 — `mid` is the last probe, not a lower bound
        mid = (l + r) / 2;
        const u64 p = occ[off + mid] >> 1;
        if (p < lo) l = mid + 1;
        else if (p > lo) r = mid - 1;
        else break;
      }
      prev_l = mid;
      for (u32 oi = (u32)mid; oi < n; ++oi) {
        const u64 rh = occ[off + oi];
        if ((rh >> 1) > win[bi].second) break;
        const bool same = ((rh ^ mhit) & 1) == 0;
        if ((same && strand == 0) || (!same && strand == 1)) hits.push_back(hit_to_candidate(k, rh, mhit));
      }
    }
    if (n >= (u32)max_seed_freq0) rep_update(k, w, (u32)(mhit >> 1), st);
  }
  std::sort(hits.begin(), hits.end());
  rep_len = st.len;
  return max_cnt;
}
static int rescue_hits(const orc_params &P, const orc_index &ix, int strand, u32 range,
                       const std::vector<Mm> &mm, const std::vector<Cand> &mate, u32 &rep_len,
                       std::vector<u64> &hits) {
  return rescue_core(ix.k, ix.w, P.max_seed_freq0, P.min_num_seeds, strand, range, mm.size(),
                     [&](size_t i, u64 &key, u64 &val, u64 &mhit) { mhit = mm[i].hit; return ix.lookup(mm[i].hash, key, val); },
                     ix.occ.data(), mate, rep_len, hits);
}

// candidate_processor.cc:345-414.
static void merge_cands(int e, std::vector<Cand> &c1, std::vector<Cand> &c2) {
  if (c1.empty()) { c1.swap(c2); return; }
  std::vector<Cand> o;
  size_t i = 0, j = 0;
  auto far = [&](u64 p) { return o.empty() || p > o.back().pos + (u64)e; };
  while (i < c1.size() && j < c2.size()) {
    if (c1[i].pos == c2[j].pos) {
      if (far(c1[i].pos)) o.push_back(c1[i].cnt > c2[j].cnt ? c1[i] : c2[j]);
      ++i; ++j;
    } else if (c1[i].pos < c2[j].pos) { if (far(c1[i].pos)) o.push_back(c1[i]); ++i; }
    else { if (far(c2[j].pos)) o.push_back(c2[j]); ++j; }
  }
  for (; i < c1.size(); ++i) if (far(c1[i].pos)) o.push_back(c1[i]);
  for (; j < c2.size(); ++j) if (far(c2[j].pos)) o.push_back(c2[j]);
  c1.swap(o);
}

// candidate_processor.cc:75-231.  Returns 1 when MAPQ must be forced to 0.
static int supplement(const orc_params &P, const orc_index &ix, ReadState rs[2]) {
  std::vector<Cand> aug[2][2];  // [mate][strand]
  int ret = 0;
  const u32 range = 2 * (u32)P.max_insert_size;
  for (int mate = 0; mate < 2; ++mate) {
    ReadState &me = rs[mate], &ot = rs[1 - mate];
    const u32 n_mm = me.mm.size();
    bool aug_flag = true;
    for (int s = 0; s < 2 && aug_flag; ++s)
      for (const Cand &c : me.cand[s])
        if (c.cnt >= n_mm / 2) { aug_flag = false; break; }
    if (!aug_flag) continue;
    me.hits[0].clear(); me.hits[1].clear();
    int pr = 0, nr = 0;
    if (!ot.cand[0].empty()) {
      pr = rescue_hits(P, ix, 1, range, me.mm, ot.cand[0], me.rep_len, me.hits[1]);
      cluster_hits(P.error_threshold, 1, n_mm, me.hits[1], aug[mate][1]);
    }
    if (!ot.cand[1].empty()) {
      nr = rescue_hits(P, ix, 0, range, me.mm, ot.cand[1], me.rep_len, me.hits[0]);
      cluster_hits(P.error_threshold, 1, n_mm, me.hits[0], aug[mate][0]);
    }
    if (((pr < 0 && nr > 0 && -pr >= nr) || (pr > 0 && nr < 0 && pr <= -nr)) &&
        me.cand[0].size() + me.cand[1].size() == 0)
      ret = 1;
  }
  for (int mate = 0; mate < 2; ++mate)
    for (int s = 0; s < 2; ++s)
      if (!aug[mate][s].empty()) merge_cands(P.error_threshold, rs[mate].cand[s], aug[mate][s]);
  return ret;
}

// candidate_processor.cc:416-484.
static void pe_filter_dir(u32 dist, const std::vector<Cand> &c1, const std::vector<Cand> &c2,
                          std::vector<Cand> &f1, std::vector<Cand> &f2) {
  u32 i1 = 0, i2 = 0, prev_end = 0;
  int un1 = 0, un2 = 0, max1 = 6, max2 = 6;
  while (i1 < c1.size() && i2 < c2.size()) {
    if (c1[i1].pos > c2[i2].pos + dist) {
      if (i2 >= prev_end && un2 < 5 && (c1[i1].pos >> 32) == (c2[i2].pos >> 32) && c2[i2].cnt >= max2) {
        f2.push_back(c2[i2]); ++un2;
      }
      ++i2;
    } else if (c2[i2].pos > c1[i1].pos + dist) {
      if (un1 < 5 && (c1[i1].pos >> 32) == (c2[i2].pos >> 32) && c1[i1].cnt >= max1) {
        f1.push_back(c1[i1]); ++un1;
      }
      ++i1;
    } else {
      f1.push_back(c1[i1]);
      if (c1[i1].cnt > max1) max1 = c1[i1].cnt;
      u32 j = i2;
      while (j < c2.size() && c2[j].pos <= c1[i1].pos + dist) {
        if (j >= prev_end) { f2.push_back(c2[j]); if (c2[j].cnt > max2) max2 = c2[j].cnt; }
        ++j;
      }
      prev_end = j;
      ++i1;
    }
  }
}

// alignment.cc:141-192.
static int banded_align(int e, const char *pat, const char *text, int L, int *end_pos) {
  u32 Peq[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 2 * e; ++i) Peq[code(pat[i])] |= (1u << i);
  const u32 hi = 1u << (2 * e);
  u32 VP = 0, VN = 0;
  int err = 0;
  for (int i = 0; i < L; ++i) {
    Peq[code(pat[i + 2 * e])] |= hi;
    u32 X = Peq[code(text[i])] | VN;
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    VN = X & HP;
    VP = HN | ~(X | HP);
    err += 1 - (int)(D0 & 1u);
    if (err > 3 * e) return e + 1;
    for (int a = 0; a < 5; ++a) Peq[a] >>= 1;
  }
  int best = err;
  *end_pos = L - 1;
  for (int i = 0; i < 2 * e; ++i) {
    err += (int)((VP >> i) & 1u);
    err -= (int)((VN >> i) & 1u);
    if (err < best || (err == best && i + 1 == e)) { best = err; *end_pos = L + i; }
  }
  return best;
}

// alignment.cc:656-718.
static void banded_traceback(int e, int min_err, const char *pat, const char *text, int L, int *start) {
  if (min_err == 0) { *start = e; return; }
  int ham = 0;
  for (int i = 0; i < L; ++i) if (pat[i + e] != text[i]) ++ham;  // raw chars, case-sensitive (:665-669)
  if (ham == min_err) { *start = e; return; }
  u32 Peq[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 2 * e; ++i) Peq[code(pat[L - 1 + 2 * e - i])] |= (1u << i);
  const u32 hi = 1u << (2 * e);
  u32 VP = 0, VN = 0;
  int err = 0;
  for (int i = 0; i < L; ++i) {
    Peq[code(pat[L - 1 - i])] |= hi;
    u32 X = Peq[code(text[L - 1 - i])] | VN;
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    VN = X & HP;
    VP = HN | ~(X | HP);
    err += 1 - (int)(D0 & 1u);
    for (int a = 0; a < 5; ++a) Peq[a] >>= 1;
  }
  *start = 2 * e;
  for (int i = 0; i < 2 * e; ++i) {
    err += (int)((VP >> i) & 1u);
    err -= (int)((VN >> i) & 1u);
    if (err == min_err) { *start = 2 * e - (1 + i); if (i + 1 == e) return; }
  }
}

// alignment.cc:197-283 — banded Myers that stops when the band-bottom error count exceeds 2e (the read may be
// chimeric); returns the best distance over the band at the stop column, the reference end offset (negated when
// the stop is "at the beginning", :277-280) and the number of read bases consumed.
static int align_dropoff(int e, const char *pat, const char *text, int L, int *end_pos, int *read_len_out) {
  u32 Peq[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 2 * e; ++i) Peq[code(pat[i])] |= (1u << i);
  const u32 hi = 1u << (2 * e);
  u32 VP = 0, VN = 0, pVP = 0, pVN = 0;
  int err = 0, perr = 0, i = 0, fail_beginning = 0;
  for (; i < L; ++i) {
    Peq[code(pat[i + 2 * e])] |= hi;
    u32 X = Peq[code(text[i])] | VN;
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    pVN = VN; pVP = VP;
    VN = X & HP;
    VP = HN | ~(X | HP);
    perr = err;
    err += 1 - (int)(D0 & 1u);
    if (err > 2 * e) { if (i < 4 * e && i < L / 2) fail_beginning = 1; break; }
    for (int a = 0; a < 5; ++a) Peq[a] >>= 1;
  }
  if (i < L) { err = perr; VN = pVN; VP = pVP; }
  const int band_start = i - 1;
  int best = err;
  *read_len_out = i;
  *end_pos = band_start;
  for (int j = 0; j < 2 * e; ++j) {
    err += (int)((VP >> j) & 1u);
    err -= (int)((VN >> j) & 1u);
    if (err < best || (err == best && j + 1 == e)) { best = err; *end_pos = band_start + 1 + j; }
  }
  if (fail_beginning || (L > 60 && *end_pos + 1 - e - best < 30)) *end_pos = -*end_pos;
  return best;
}
// alignment.cc:285-376 — the same from the 3' end (used for the reverse-complement strand).
static int align_dropoff_3end(int e, const char *pat, const char *text, int L, int *end_pos, int *read_len_out) {
  u32 Peq[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 2 * e; ++i) Peq[code(pat[L + 2 * e - 1 - i])] |= (1u << i);
  const u32 hi = 1u << (2 * e);
  u32 VP = 0, VN = 0, pVP = 0, pVN = 0;
  int err = 0, perr = 0, i = 0, fail_beginning = 0;
  for (; i < L; ++i) {
    Peq[code(pat[L - 1 - i])] |= hi;
    u32 X = Peq[code(text[L - 1 - i])] | VN;
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    pVN = VN; pVP = VP;
    VN = X & HP;
    VP = HN | ~(X | HP);
    perr = err;
    err += 1 - (int)(D0 & 1u);
    if (err > 2 * e) { if (i < 4 * e && i < L / 2) fail_beginning = 1; break; }
    for (int a = 0; a < 5; ++a) Peq[a] >>= 1;
  }
  if (i < L) { err = perr; VN = pVN; VP = pVP; }
  const int band_start = i - 1;
  int best = err;
  *read_len_out = i;
  *end_pos = band_start;
  for (int j = 0; j < 2 * e; ++j) {
    err += (int)((VP >> j) & 1u);
    err -= (int)((VN >> j) & 1u);
    if (err < best || (err == best && j + 1 == e)) { best = err; *end_pos = band_start + (1 + j); }
  }
  if (fail_beginning || (L > 60 && *end_pos + 1 - e - best < 30)) *end_pos = -*end_pos;
  return best;
}
// alignment.cc:24-83 (n_cigar == 0 on the BED/pairs path): extend an exact match into the skipped 5' gap.
// `ref` is the whole reference sequence (NUL padded), `read` NUL terminated.
static int adjust_gap_beginning(int strand, const char *ref, const char *read, int *gap, int read_end, int ref_start, int ref_end) {
  int i, j;
  if (strand == 0) {
    if (*gap <= 0) return ref_start;
    for (i = *gap - 1, j = ref_start - 1; i >= 0 && j >= 0; --i, --j)
      if (read[i] != ref[j] && read[i] != ref[j] - 'a' + 'A') break;
    *gap = i + 1;
    return j + 1;
  }
  if (*gap <= 0) return ref_end;
  for (i = read_end + 1, j = ref_end + 1; read[i] && ref[j]; ++i, ++j)
    if (read[i] != ref[j] && read[i] != ref[j] - 'a' + 'A') break;
  *gap = *gap + i - (read_end + 1);
  return j - 1;
}

static inline bool valid_cand(int e, u32 ref_len, u32 pos, u32 L) {  // draft_mapping_generator.cc:59-70
  return !(pos < (u32)e || pos >= ref_len || pos + L + (u32)e >= ref_len);
}
static inline void tally(ReadState &rs, int err) {  // the best/second-best bookkeeping, :217-230 etc.
  if (err < rs.min_err) { rs.second_min_err = rs.min_err; rs.n_second_best = rs.n_best; rs.min_err = err; rs.n_best = 1; }
  else if (err == rs.min_err) rs.n_best++;
  else if (err == rs.second_min_err) rs.n_second_best++;
  else if (err < rs.second_min_err) { rs.n_second_best = 1; rs.second_min_err = err; }
}

// draft_mapping_generator.cc:9-57 (non-split), with :72-157 fast path, :159-357 lane-group driver and
// :359-557 per-candidate driver.  The SSE kernels agree with the scalar routine on accept/reject,
// distance and end position (SURVEY.md §2.2), so groups are replayed with the scalar routine.
static void verify_read(const orc_params &P, const orc_reference &ref, const char *read,
                        const std::string &neg, u32 L, ReadState &rs) {
  const int e = P.error_threshold;
  rs.min_err = e + 1; rs.n_best = 0; rs.second_min_err = e + 1; rs.n_second_best = 0;
  // fast path: exactly one candidate overall and it is supported by all minimizers
  if (rs.cand[0].size() + rs.cand[1].size() == 1) {
    int n_all = 0, idx = 0, strand = 0;
    for (size_t i = 0; i < rs.cand[0].size(); ++i) if (rs.cand[0][i].cnt == rs.mm.size()) { idx = i; ++n_all; }
    for (size_t i = 0; i < rs.cand[1].size(); ++i) if (rs.cand[1][i].cnt == rs.mm.size()) { idx = i; strand = 1; ++n_all; }
    if (n_all == 1) {
      rs.min_err = 0; rs.n_best = 1; rs.n_second_best = 0;  // set before the validity check (:113-115)
      const Cand &c = rs.cand[strand][idx];
      const u32 rid = (u32)(c.pos >> 32);
      const u32 pos = strand == 0 ? (u32)c.pos : (u32)c.pos - L + 1;
      if (valid_cand(e, ref.lens[rid], pos, L)) {
        rs.map[strand].push_back({0, strand == 0 ? c.pos + L - 1 : c.pos});
        return;
      }
    }
  }
  std::sort(rs.cand[0].begin(), rs.cand[0].end(), cand_less);
  std::sort(rs.cand[1].begin(), rs.cand[1].end(), cand_less);
  const int lanes = e < 8 ? 8 : (e < 16 ? 4 : 0);  // mapping_parameters.h:80-88
  for (int s = 0; s < 2; ++s) {
    const std::vector<Cand> &cs = rs.cand[s];
    const char *text = s == 0 ? read : neg.data();
    auto run_one = [&](const Cand &c, bool &failed) {
      const u32 rid = (u32)(c.pos >> 32);
      const u32 pos = s == 0 ? (u32)c.pos : (u32)c.pos - L + 1;
      int endp = 0;
      const int err = banded_align(e, ref.seqs[rid].data() + pos - e, text, L, &endp);
      failed = err > e;
      if (!failed) {
        tally(rs, err);
        rs.map[s].push_back({err, s == 0 ? c.pos - e + endp : c.pos - L + 1 - e + endp});
      }
    };
    if (cs.size() < (size_t)lanes) {
      for (const Cand &c : cs) {
        const u32 pos = s == 0 ? (u32)c.pos : (u32)c.pos - L + 1;
        if (!valid_cand(e, ref.lens[(u32)(c.pos >> 32)], pos, L)) continue;
        bool f; run_one(c, f);
      }
      continue;
    }
    std::vector<Cand> group;
    u32 threshold = 0;
    size_t ci = 0;
    while (ci < cs.size()) {
      if (cs[ci].cnt < threshold) break;
      const u32 pos = s == 0 ? (u32)cs[ci].pos : (u32)cs[ci].pos - L + 1;
      if (!valid_cand(e, ref.lens[(u32)(cs[ci].pos >> 32)], pos, L)) { ++ci; continue; }
      group.push_back(cs[ci]); ++ci;
      if ((int)group.size() < lanes) continue;
      for (const Cand &c : group) { bool f; run_one(c, f); if (f) threshold = c.cnt; }
      group.clear();
    }
    for (const Cand &c : group) { bool f; run_one(c, f); }
  }
}

// draft_mapping_generator.cc:9-57 + :359-557 with --split-alignment: per-candidate scalar driver, drop-off
// alignment, optional skip of the first 20-e read bases, num_errors := -(matched length), count-threshold pruning.
static void verify_read_split(const orc_params &P, const orc_reference &ref, const char *read, const std::string &neg, u32 L, ReadState &rs) {
  const int e = P.error_threshold;
  rs.min_err = e + 1; rs.n_best = 0; rs.second_min_err = e + 1; rs.n_second_best = 0;
  std::sort(rs.cand[0].begin(), rs.cand[0].end(), cand_less);
  std::sort(rs.cand[1].begin(), rs.cand[1].end(), cand_less);
  for (int s = 0; s < 2; ++s) {
    const std::vector<Cand> &cs = rs.cand[s];
    u32 threshold = 0;
    for (size_t ci = 0; ci < cs.size(); ++ci) {
      if (cs[ci].cnt < threshold) break;
      const u32 rid = (u32)(cs[ci].pos >> 32);
      const u32 pos = s == 0 ? (u32)cs[ci].pos : (u32)cs[ci].pos - L + 1;
      if (!valid_cand(e, ref.lens[rid], pos, L)) continue;
      int endp = L, gap = 0, nerr = 0, actual = 0, rml = 0;
      const int allow_gap = 20 - e;
      const char *win = ref.seqs[rid].data() + pos - e;
      if (s == 0) {
        nerr = align_dropoff(e, win, read, L, &endp, &rml);
        if (endp < 0 && allow_gap > 0) {
          const int b_err = nerr, b_end = -endp, b_rml = rml;
          nerr = align_dropoff(e, win + allow_gap, read + allow_gap, L - allow_gap, &endp, &rml);
          if (nerr > e || endp < 0) { nerr = b_err; endp = b_end; rml = b_rml; }
          else { gap = allow_gap; endp += gap; rml += gap; }
        }
      } else {
        nerr = align_dropoff_3end(e, win, neg.data(), L, &endp, &rml);
        if (endp < 0 && allow_gap > 0) {
          const int b_err = nerr, b_end = -endp, b_rml = rml;
          nerr = align_dropoff_3end(e, win, neg.data(), L - allow_gap, &endp, &rml);
          if (nerr > e || endp < 0) { nerr = b_err; endp = b_end; rml = b_rml; }
          else { gap = allow_gap; endp += gap; rml += gap; }
        }
      }
      if (endp + 1 - e - nerr - gap >= 30) { actual = nerr; nerr = -(endp - e - nerr - gap); }
      else { nerr = e + 1; actual = e + 1; }
      // (GetLongestMatchLength, :474-483, only feeds a comparison between two per-iteration locals that are both
      //  zero-initialised inside this loop — it cannot change anything)
      if (nerr <= e) {
        if (nerr < rs.min_err) {
          rs.second_min_err = rs.min_err; rs.n_second_best = rs.n_best; rs.min_err = nerr; rs.n_best = 1;
          threshold = cs.size() > 50 ? cs[ci].cnt : cs[ci].cnt / 2;
        } else if (nerr == rs.min_err) rs.n_best++;
        else if (nerr == rs.second_min_err) rs.n_second_best++;
        else if (nerr < rs.second_min_err) { rs.n_second_best = 1; rs.second_min_err = nerr; }
        rs.map[s].push_back({nerr, s == 0 ? cs[ci].pos - e + endp : cs[ci].pos - gap});
        rs.split[s].push_back(((actual & 0xff) << 24) | ((gap & 0xff) << 16) | (rml & 0xffff));
      }
    }
  }
}

struct PairState {
  int min_sum, second_min_sum, n_best, n_second_best;
  std::vector<std::pair<u32, u32>> best[4];  // [0]=F1R2, [1]=F2R1, [2]=F1F2, [3]=R1R2 (paired_end_mapping_metadata.h:66-98)
};

// mapping_generator.h:346-484 (non-split branch).
static void pair_dir(const orc_params &P, int s1, u32 L1, u32 L2, const std::vector<Draft> &m1,
                     const std::vector<Draft> &m2, PairState &ps, std::vector<std::pair<u32, u32>> &best) {
  u32 i1 = 0, i2 = 0;
  const u64 ins = P.max_insert_size, ovl = P.min_read_length;
  while (i1 < m1.size() && i2 < m2.size()) {
    if ((s1 == 1 && m1[i1].pos > m2[i2].pos + ins - L2) || (s1 == 0 && m1[i1].pos > m2[i2].pos + L1 - ovl)) ++i2;
    else if ((s1 == 0 && m2[i2].pos > m1[i1].pos + ins - L1) || (s1 == 1 && m2[i2].pos > m1[i1].pos + L2 - ovl)) ++i1;
    else {
      u32 j = i2;
      while (j < m2.size() && ((s1 == 0 && m2[j].pos <= m1[i1].pos + ins - L1) ||
                               (s1 == 1 && m2[j].pos <= m1[i1].pos + L2 - ovl))) {
        const int sum = m1[i1].err + m2[j].err;
        if (sum < ps.min_sum) {
          ps.second_min_sum = ps.min_sum; ps.n_second_best = ps.n_best; ps.min_sum = sum; ps.n_best = 1;
          best.clear(); best.push_back({i1, j});
        } else if (sum == ps.min_sum) { ps.n_best++; best.push_back({i1, j}); }
        else if (sum == ps.second_min_sum) ps.n_second_best++;
        else if (sum < ps.second_min_sum) { ps.second_min_sum = sum; ps.n_second_best = 1; }
        ++j;
      }
      ++i1;
    }
  }
}

// mapping_generator.h:920-1022 (non-split).
static uint8_t mapq_se(int num_errors, uint16_t aln_len, int read_len, int max_diff, const ReadState &rs) {
  const int coef_len = 50;
  const int coef_frac = log(coef_len);  // == 3 (:925)
  aln_len = aln_len > read_len ? aln_len : read_len;
  const double ident = 1 - (double)num_errors / aln_len;
  int mapq = 0;
  int second = rs.second_min_err;
  if (rs.n_best > 1) {
  } else {
    if (second > num_errors + max_diff) second = num_errors + max_diff;
    double tmp = aln_len < coef_len ? 1.0 : coef_frac / log(aln_len);
    tmp *= ident * ident;
    mapq = 5 * 6.02 * (second - num_errors) * tmp * tmp + 0.499;
  }
  if (rs.n_second_best > 0) mapq -= (int)(4.343 * log(rs.n_second_best + 1) + 0.499);
  if (mapq > 60) mapq = 60;
  if (mapq < 0) mapq = 0;
  if (rs.rep_len > 0) {
    double frac = rs.rep_len / (double)read_len;
    if (rs.rep_len >= (u32)read_len) frac = 0.999;
    if (ident <= 0.95) mapq = mapq * (1 - sqrt(frac)) + 0.499;
    else if (ident <= 0.97) mapq = mapq * (1 - frac) + 0.499;
    else if (ident >= 0.999) mapq = mapq * (1 - frac * frac * frac * frac) + 0.499;
    else mapq = mapq * (1 - frac * frac) + 0.499;
  }
  return (uint8_t)mapq;
}

#define ORC_RAW_MAPQ(diff, a) ((int)(5 * 6.02 * (diff) / (a) + .499))
// mapping_generator.h:1027-1192 (non-split).
static uint8_t mapq_pe(int e1, int e2, uint16_t al1, uint16_t al2, int L1, int L2, int force,
                       const PairState &ps, const ReadState rs[2], uint8_t *mapq1_out = nullptr, uint8_t *mapq2_out = nullptr) {
  uint8_t pe = 0;
  const int unpaired = rs[0].min_err + rs[1].min_err + 3;
  if (ps.n_best <= 1) {
    const int adj = ps.second_min_sum < unpaired ? ps.second_min_sum : unpaired;
    pe = ORC_RAW_MAPQ(adj - ps.min_sum, 1);
    if (ps.n_second_best > 0) pe -= (int)(4.343 * log(ps.n_second_best + 1) + 0.499);  // uint8 wrap (:1073)
    if (pe > 60) pe = 60;
    const int rep = rs[0].rep_len + rs[1].rep_len;
    if (rep > 0) {
      const double total = L1 + L2;
      double frac = (double)rep / total;
      if (rep >= total) frac = 0.999;
      const double id1 = 1 - (double)e1 / (L1 > al1 ? L1 : al1);
      const double id2 = 1 - (double)e2 / (L2 > al2 ? L2 : al2);
      const double ident = id1 < id2 ? id1 : id2;
      if (ident <= 0.95) pe = pe * (1 - sqrt(frac)) + 0.499;
      else if (ident <= 0.97) pe = pe * (1 - frac) + 0.499;
      else if (ident >= 0.999) pe = pe * (1 - frac * frac * frac * frac) + 0.499;
      else pe = pe * (1 - frac * frac) + 0.499;
    }
  }
  uint8_t q1 = mapq_se(e1, al1, L1, 2, rs[0]);
  uint8_t q2 = mapq_se(e2, al2, L2, 2, rs[1]);
  q1 = q1 > pe ? q1 : pe < q1 + pe * 0.65 ? pe : q1 + pe * 0.65;
  q2 = q2 > pe ? q2 : pe < q2 + pe * 0.65 ? pe : q2 + pe * 0.65;
  q1 *= 1.2; if (q1 > 60) q1 = 60;
  q2 *= 1.2; if (q2 > 60) q2 = 60;
  if (mapq1_out) *mapq1_out = q1;
  if (mapq2_out) *mapq2_out = q2;
  uint8_t q = q1 < q2 ? q1 : q2;
  if (q < 60 && force >= 0 && force < q) q = force;
  return q;
}

// mapping_generator.h:657-917, BED branch, non-split: start from traceback, end = draft end.
static void ref_span(const orc_params &P, const orc_reference &ref, const Draft &d, const char *read_seq,
                     int L, u32 &start, u32 &end) {
  const int e = P.error_threshold;
  const u32 rid = (u32)(d.pos >> 32), rp = (u32)d.pos;
  u32 vws = rp + 1 > (u32)(L + e) ? rp + 1 - L - e : 0;
  if (rp + e >= ref.lens[rid]) vws = ref.lens[rid] - e - L;
  int s = 0;
  banded_traceback(e, d.err, ref.seqs[rid].data() + vws, read_seq, L, &s);
  start = vws + s;
  end = rp;
}

// mapping_generator.h:389-415 — split alignment pairs every best mapping of mate 1 with every best mapping of mate 2.
static void pair_dir_split(const ReadState rs[2], int s1, int s2, PairState &ps, std::vector<std::pair<u32, u32>> &best) {
  const std::vector<Draft> &m1 = rs[0].map[s1], &m2 = rs[1].map[s2];
  if (m1.empty() || m2.empty()) return;
  for (u32 i1 = 0; i1 < m1.size(); ++i1) {
    if (m1[i1].err != rs[0].min_err) continue;
    for (u32 i2 = 0; i2 < m2.size(); ++i2) {
      if (m2[i2].err != rs[1].min_err) continue;
      best.push_back({i1, i2});
      ps.min_sum = rs[0].min_err + rs[1].min_err;
      ps.n_best++;
    }
  }
}

// mapping_generator.h:920-1022 with split_alignment (num_errors = -(matched length)).
static uint8_t mapq_se_split(const orc_params &P, int strand, int num_errors, uint16_t aln_len, int read_len, int max_diff, const ReadState &rs) {
  const int coef_len = 50;
  const int coef_frac = log(coef_len);
  double ident = 1 - (double)num_errors / aln_len;
  ident = (double)(-num_errors) / aln_len;
  if (ident > 1) ident = 1;
  int mapq = 0;
  int second = rs.second_min_err;
  if (rs.n_best > 1) {
  } else {
    if (second > num_errors + max_diff) second = num_errors + max_diff;
    double tmp = aln_len < coef_len ? 1.0 : coef_frac / log(aln_len);
    tmp *= ident * ident;
    mapq = 5 * 6.02 * (second - num_errors) * tmp * tmp + 0.499;
  }
  if (rs.n_second_best > 0) mapq -= (int)(4.343 * log(rs.n_second_best + 1) + 0.499);
  if (mapq > 60) mapq = 60;
  if (mapq < 0) mapq = 0;
  if (rs.rep_len > 0) {
    double frac = rs.rep_len / (double)read_len;
    if (rs.rep_len >= (u32)read_len) frac = 0.999;
    if (ident <= 0.95) mapq = mapq * (1 - sqrt(frac)) + 0.499;
    else if (ident <= 0.97) mapq = mapq * (1 - frac) + 0.499;
    else if (ident >= 0.999) mapq = mapq * (1 - frac * frac * frac * frac) + 0.499;
    else mapq = mapq * (1 - frac * frac) + 0.499;
  }
  if (aln_len < read_len - P.error_threshold && second != num_errors) {
    if (rs.rep_len >= aln_len && rs.rep_len < (u32)read_len && aln_len < read_len / 3) mapq = 0;
    const int diff = second - num_errors;
    const u32 num_candidates = rs.cand[strand].size();
    if (second - num_errors <= P.error_threshold * 3 / 4 && num_candidates >= 5) mapq -= (num_candidates / 5 / diff);
    if (mapq < 0) mapq = 0;
    if (rs.n_second_best > 0 && second - num_errors <= P.error_threshold * 3 / 4) mapq /= (rs.n_second_best / diff + 1);
  }
  return (uint8_t)mapq;
}

// mapping_generator.h:657-917, BED/pairs branch with split_alignment.
static void ref_span_split(const orc_params &P, const orc_reference &ref, const Draft &d, int strand, int split_word, const char *read_seq,
                           int full_len, u32 &start, u32 &end) {
  const int e = P.error_threshold;
  const u32 rid = (u32)(d.pos >> 32), rp = (u32)d.pos;
  const int split_site = split_word & 0xffff;
  int gap = (split_word >> 16) & 0xff;
  const int actual = (split_word >> 24) & 0xff;
  int L = split_site - gap;
  u32 vws = rp + 1 > (u32)(L + e) ? rp + 1 - L - e : 0;
  if (rp + e >= ref.lens[rid]) vws = ref.lens[rid] - e - L;
  const char *rseq = ref.seqs[rid].data();
  if (strand == 0) {
    int s = 0;
    banded_traceback(e, actual, rseq + vws, read_seq + gap, L, &s);
    if (gap > 0) s = adjust_gap_beginning(0, rseq, read_seq, &gap, L - 1, vws + s, rp) - vws;
    start = vws + s;
    end = rp;
    return;
  }
  const int read_start_site = full_len - split_site;
  int s = e, en = rp - vws + 1;
  banded_align(e, rseq + vws, read_seq + read_start_site, L, &en);
  en += 1;
  if (gap > 0) en = adjust_gap_beginning(1, rseq, read_seq + read_start_site, &gap, L - 1, vws + s, vws + en) - vws + 1;
  start = vws + s;
  end = vws + en - 1;
}

// ----------------------------------------------------------------------------------------------
// Cell barcodes: 2-bit packing (utils.h:107-126, N -> A), whitelist + abundance (chromap.cc:388-548),
// correction (chromap.cc:572-799).
static u64 barcode_seed(const char *s, u32 len) {
  u64 seed = 0;
  for (u32 i = 0; i < len; ++i) { const uint8_t b = code(s[i]); seed = b < 4 ? (seed << 2) | b : seed << 2; }
  return seed;
}
struct orc_whitelist {
  std::vector<u64> keys;    // sorted
  std::vector<u32> counts;  // abundance in the sampled barcodes
  u64 num_sample = 0;
  u32 bc_len = 0;
  int find(u64 k) const {
    auto it = std::lower_bound(keys.begin(), keys.end(), k);
    return (it != keys.end() && *it == k) ? (int)(it - keys.begin()) : -1;
  }
};
struct BcCand {
  u32 idx1; char b1; u32 idx2; char b2; double score;
  bool operator>(const BcCand &o) const {  // utils.h:23-35
    return std::tie(score, idx1, b1, idx2, b2) > std::tie(o.score, o.idx1, o.b1, o.idx2, o.b2);
  }
};
// chromap.cc:572-799.  Returns true if the (possibly corrected, in place) barcode is in the whitelist.
static bool correct_barcode(const orc_whitelist &wl, int err_threshold, double prob_threshold, char *bc, const char *qual, u32 len,
                            u64 *n_in_whitelist, u64 *n_corrected) {
  const u64 key = barcode_seed(bc, len);
  std::vector<int> npos;  // little endian: from the right end (sequence_batch.h:85-104)
  for (int i = (int)len - 1; i >= 0; --i) if (bc[i] == 'N') npos.push_back(len - 1 - i);
  if (npos.size() > (size_t)err_threshold) return false;
  if (npos.empty() && wl.find(key) >= 0) { ++*n_in_whitelist; return true; }
  if (err_threshold <= 0) return false;
  static const char tab[4] = {'A', 'C', 'G', 'T'};
  std::vector<BcCand> cands;
  const u64 mask = 3;
  u32 i_start = 0, i_end = len, ti_limit = 3;
  if (!npos.empty()) { i_start = npos[0]; i_end = npos[0] + 1; ti_limit = 4; }
  for (u32 i = i_start; i < i_end; ++i) {
    const u64 keep = ~(mask << (2 * i)) & key;
    u64 b1 = (key >> (2 * i)) & mask;
    for (u32 ti = 0; ti < ti_limit; ++ti) {
      b1 = (b1 + 1) & mask;
      const u64 k1 = keep | (b1 << (2 * i));
      int f = wl.find(k1);
      if (f >= 0) {
        const double abundance = wl.counts[f] / (double)wl.num_sample;
        int q = qual[len - 1 - i] - 33;
        q = q > 40 ? 40 : q; q = q < 3 ? 3 : q;
        cands.push_back({len - 1 - i, tab[b1], 0, 0, pow(10.0, ((-q) / 10.0)) * abundance});
      }
      if (err_threshold == 2) {
        u32 j_start = i + 1, j_end = len, ti2_limit = 3;
        if (npos.size() == 2) { j_start = npos[1]; j_end = npos[1] + 1; ti2_limit = 4; }
        for (u32 j = j_start; j < j_end; ++j) {
          const u64 keep2 = ~(mask << (2 * j)) & k1;
          u64 b2 = (k1 >> (2 * j)) & mask;
          for (u32 t2 = 0; t2 < ti2_limit; ++t2) {
            b2 = (b2 + 1) & mask;
            const u64 k2 = keep2 | (b2 << (2 * j));
            f = wl.find(k2);
            if (f >= 0) {
              const double abundance = wl.counts[f] / (double)wl.num_sample;
              int q = qual[len - 1 - j] - 33;
              q = q > 40 ? 40 : q; q = q < 3 ? 3 : q;
              int q1 = qual[len - 1 - i] - 33;
              q1 = q1 > 40 ? 40 : q1; q1 = q1 < 3 ? 3 : q1;
              q += q1;
              cands.push_back({len - 1 - i, tab[b1], len - 1 - j, tab[b2], pow(10.0, ((-q) / 10.0)) * abundance});
            }
          }
        }
      }
    }
  }
  if (cands.empty()) return false;
  size_t best = 0;
  if (cands.size() > 1) {
    std::sort(cands.begin(), cands.end(), std::greater<BcCand>());
    double sum = 0;
    for (const BcCand &c : cands) sum += c.score;
    if (!(cands[0].score / sum > prob_threshold)) return false;
  }
  bc[cands[best].idx1] = cands[best].b1;
  if (cands[best].b2 != 0) bc[cands[best].idx2] = cands[best].b2;
  ++*n_corrected;
  return true;
}

static const bool g_debug = getenv("ORC_DEBUG") != nullptr;
struct orc_mapper {
  orc_params P;
  const orc_index *ix;
  const orc_reference *ref;
  const orc_whitelist *wl = nullptr;  // scATAC: barcode whitelist with abundances (may stay null: barcodes used as they are)
  int bc_err_threshold = 1;           // --bc-error-threshold (mapping_parameters.h:43)
  double bc_prob_threshold = 0.9;     // --bc-probability-threshold
  int output_not_in_whitelist = 0;    // --output-mappings-not-in-whitelist
};

static void revcomp(const char *s, u32 L, std::string &out) {  // sequence_batch.h:123-134
  static const char tab[8] = {'A', 'C', 'G', 'T', 'N', 'N', 'N', 'N'};
  out.resize(L);
  for (u32 i = 0; i < L; ++i) out[i] = tab[(uint8_t)3 ^ code(s[L - 1 - i])];
}

// chromap.cc:176-289.  Works on copies; returns trimmed lengths.  neg strings are trimmed from the front.
static void trim_adapters(const orc_params &P, std::string &r1, std::string &r2, std::string &n1, std::string &n2) {
  const u32 raw1 = r1.size(), raw2 = r2.size();
  const bool swap = !(raw1 <= raw2);
  const char *read1 = swap ? r2.data() : r1.data();
  const std::string &neg2 = swap ? n1 : n2;
  const u32 L1 = swap ? raw2 : raw1, L2 = swap ? raw1 : raw2;
  const int min_ovl = P.min_read_length, seed = min_ovl / 2, max_err = 1;
  for (int si = 0; si < max_err + 1; ++si) {
    size_t sp = neg2.find(read1 + si * seed, 0, seed);
    while (sp != std::string::npos) {
      const bool before_ok = sp >= (size_t)(si * seed);
      const bool ovl_ok = (int)(L2 - sp + seed * si) >= min_ovl;
      if (!before_ok || !ovl_ok) { sp = neg2.find(read1 + si * seed, sp + 1, seed); continue; }
      bool ok = true;
      int ne = 0;
      for (int i = 0; i < seed * si; ++i) {
        if (neg2[sp - si * seed + i] != read1[i]) ++ne;
        if (ne > max_err) { ok = false; break; }
      }
      for (u32 i = seed; i + sp < L2 && si * seed + i < L1; ++i) {
        if (neg2[sp + i] != read1[si * seed + i]) ++ne;
        if (ne > max_err) { ok = false; break; }
      }
      if (ok) {
        int ovl = L2 - sp + si * seed, off2 = 0;
        if (ovl > (int)L1) { off2 = ovl - L1; ovl = L1; }
        const int t1 = swap ? ovl + off2 : ovl, t2 = swap ? ovl : ovl + off2;
        auto trim = [](std::string &r, std::string &n, int len) {  // sequence_batch.h:136-151
          if (len >= (int)r.size()) return;
          n.erase(0, r.size() - len);
          r.resize(len);
        };
        trim(r1, n1, t1);
        trim(r2, n2, t2);
        return;
      }
      sp = neg2.find(read1 + si * seed, sp + 1, seed);
    }
  }
}

// One iteration of the taskloop, chromap.h:892-1143 (bulk data, BED, non-split).
// ---- SAM output (round-2 groundwork: the oracle side of SURVEY.md 8f rank 3; the CUDA path does not emit SAM yet) ------
// Semi-global affine alignment of the read (outer loop) against a reference window (banded, band w, one direction byte
// per cell, traceback to a CIGAR) with the arithmetic and tie rules of ksw_semi_global3 (ksw.cc:505-626): the read may
// start anywhere in the first w window positions for free and end at the best of the last w.
struct SamAln { std::vector<u32> cigar; int start = 0, end = 0, score = 0; };
static void sg_align(const char *win, int wlen, const char *read, int rlen, int match, int mismatch, int o_del, int e_del, int o_ins, int e_ins, int w,
                     SamAln &out) {
  const int NEG = -0x40000000;
  auto sc = [&](char a, char b) { const int x = code(a), y = code(b); return (x < 4 && y < 4) ? (x == y ? match : -mismatch) : 0; };  // mapping_generator.h:661-670
  const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
  const int n_col = wlen < 2 * w + 1 ? wlen : 2 * w + 1;
  std::vector<uint8_t> z((size_t)n_col * rlen, 0);
  std::vector<int> H(wlen + 1), E(wlen + 1);
  H[0] = 0; E[0] = NEG;
  int j = 1;
  for (; j <= wlen && j <= w; ++j) { H[j] = 0; E[j] = NEG; }
  for (; j <= wlen; ++j) H[j] = E[j] = NEG;
  for (int i = 0; i < rlen; ++i) {
    int f = NEG;
    const int beg = i, end = i + w + 1 < wlen ? i + w + 1 : wlen;
    int h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : NEG;
    uint8_t *zi = &z[(size_t)i * n_col];
    for (j = beg; j < end; ++j) {
      int m = H[j], e = E[j];
      H[j] = h1;
      m += sc(read[i], win[j]);
      uint8_t d = m >= e ? 0 : 1;
      int h = m >= e ? m : e;
      d = h >= f ? d : 2;
      h = h >= f ? h : f;
      h1 = h;
      int t = m - oe_del;
      e -= e_del;
      if (e > t) d |= 1 << 2; else e = t;
      E[j] = e;
      t = m - oe_ins;
      f -= e_ins;
      if (f > t) d |= 2 << 4; else f = t;
      zi[j - beg] = d;
    }
    H[end] = h1; E[end] = NEG;
  }
  int score = H[wlen], best = wlen;
  for (j = 1; j < w; ++j) if (H[wlen - j] > score) { score = H[wlen - j]; best = wlen - j; }
  out.score = score; out.end = best;
  std::vector<std::pair<int, int>> ops;  // (op, len) from the end
  auto push = [&](int op, int len) { if (!ops.empty() && ops.back().first == op) ops.back().second += len; else ops.push_back({op, len}); };
  int i = rlen - 1, k = best - 1, which = 0;
  while (i >= 0 && k >= 0) {
    which = z[(size_t)i * n_col + (k - i)] >> (which << 1) & 3;
    if (which == 0) { push(0, 1); --i; --k; }
    else if (which == 1) { push(1, 1); --i; }
    else { push(2, 1); --k; }
  }
  if (i >= 0) push(1, i + 1);
  out.start = k + 1;
  out.cigar.clear();
  for (size_t q = ops.size(); q-- > 0;) out.cigar.push_back((u32)ops[q].second << 4 | (u32)ops[q].first);
}

struct SamRec {  // SAMMapping (sam_mapping.h), bulk data
  u32 read_id; std::string name; int64_t pos; int rid; int64_t mpos; int mrid; int tlen; int flag; int strand_pos; int is_unique; int mapq; int nm;
  std::vector<u32> cigar; std::string md, seq, qual;
};

// GetRefStartEndPositionForReadFromMapping, SAM branch, non-split (mapping_generator.h:696-760,807-855) + GenerateNMAndMDTag
// (alignment.cc:85-139).  read_seq is the strand's sequence (the reverse complement for the - strand).
static void ref_span_sam(const orc_params &P, const orc_reference &ref, const Draft &d, const char *read_seq, int L, u32 &start, u32 &end, SamRec &r) {
  const int e = P.error_threshold;
  const u32 rid = (u32)(d.pos >> 32), rp = (u32)d.pos;
  u32 vws = rp + 1 > (u32)(L + e) ? rp + 1 - L - e : 0;
  if (rp + e >= ref.lens[rid]) vws = ref.lens[rid] - e - L;
  const char *rseq = ref.seqs[rid].data();
  SamAln a;
  sg_align(rseq + vws, L + 2 * e, read_seq, L, 1, 4, 6, 1, 6, 1, 2 * e + 1, a);  // mapping_parameters.h:20-23 defaults
  start = vws + a.start;
  end = vws + a.end - 1;
  r.cigar = a.cigar;
  r.nm = 0; r.md.clear();
  int nmatch = 0, rpos = 0, gpos = 0;
  const char *g = rseq + start;
  for (u32 c : a.cigar) {
    const int op = c & 0xf, len = c >> 4;
    if (op == 0) {
      for (int q = 0; q < len; ++q, ++rpos, ++gpos) {
        if (g[gpos] == read_seq[rpos] || g[gpos] - 'a' + 'A' == read_seq[rpos]) ++nmatch;
        else { ++r.nm; r.md += std::to_string(nmatch); nmatch = 0; r.md.push_back(g[gpos]); }
      }
    } else if (op == 1) { r.nm += len; rpos += len; }
    else { r.nm += len; r.md += std::to_string(nmatch); nmatch = 0; r.md.push_back('^'); for (int q = 0; q < len; ++q) r.md.push_back(g[gpos++]); }
  }
  r.md += std::to_string(nmatch);
}

struct PafRec {  // PAFMapping / PairedPAFMapping (paf_mapping.h) as the reference FILLS them: EmplaceBackPairedEndMappingRecord
  // (mapping_generator.cc:146-167) passes (start, negative alignment length, fragment length, positive alignment length) to a
  // constructor that takes (start, fragment length, positive alignment length, negative alignment length) -- kept as it is.
  u32 read_id, rid, start; std::string name1, name2; uint16_t len1, len2, frag, pal, nal; uint8_t mapq, mapq1, mapq2, dir, uniq, dups;
};
struct SamSink { std::vector<SamRec> *recs; const char *name1, *qual1, *name2, *qual2; std::vector<PafRec> *paf = nullptr; };

// The part of the taskloop body after verification (chromap.h:1099-1143): SortMappingsByPositions, best pairs, sampling,
// spans, MAPQ, records.  Separate from map_one_pair so that tests can enter it with prepared draft mappings (orc_emit_test).
static int finish_pair(const orc_params &P, const orc_reference &ref, std::mt19937 &gen, const std::string r[2], const std::string neg[2],
                       const u32 L[2], ReadState rs[2], int sup, u32 read_id, orc_pe_record *out, int cap, orc_pair_trace *tr,
                       const SamSink *sam) {
  if (rs[0].map[0].size() + rs[0].map[1].size() == 0 || rs[1].map[0].size() + rs[1].map[1].size() == 0) return 0;
  // mapping_metadata.h:70-78 sorts by position only; equal positions are interchangeable for the
  // output (the lower-error one is the only one that can be in a best pair), so (pos, err) is used.
  auto by_pos = [](const Draft &a, const Draft &b) { return a.pos != b.pos ? a.pos < b.pos : a.err < b.err; };
  if (!P.split_alignment)  // chromap.h:1099-1106: split alignment keeps verification order (mappings stay aligned with split sites)
    for (int m = 0; m < 2; ++m) for (int s = 0; s < 2; ++s) std::sort(rs[m].map[s].begin(), rs[m].map[s].end(), by_pos);
  const int force = sup != 0 ? 0 : -1;
  // mapping_generator.h:160-253
  PairState ps;
  ps.min_sum = 2 * P.error_threshold + 1; ps.n_best = 0; ps.second_min_sum = ps.min_sum; ps.n_second_best = 0;
  if (P.split_alignment) {
    pair_dir_split(rs, 0, 1, ps, ps.best[0]);
    pair_dir_split(rs, 1, 0, ps, ps.best[1]);
    pair_dir_split(rs, 0, 0, ps, ps.best[2]);
    pair_dir_split(rs, 1, 1, ps, ps.best[3]);
  } else {
    pair_dir(P, 0, L[0], L[1], rs[0].map[0], rs[1].map[1], ps, ps.best[0]);
    pair_dir(P, 1, L[0], L[1], rs[0].map[1], rs[1].map[0], ps, ps.best[1]);
  }
  if (tr) { tr->min_sum_errors = ps.min_sum; tr->second_min_sum_errors = ps.second_min_sum; tr->n_best_pairs = ps.n_best; tr->n_second_best_pairs = ps.n_second_best; }
  if (ps.n_best > P.drop_repetitive_reads) return 0;
  std::vector<int> sel(P.max_num_best_mappings);
  std::iota(sel.begin(), sel.end(), 0);
  if (ps.n_best > P.max_num_best_mappings) {
    for (int i = P.max_num_best_mappings; i < ps.n_best; ++i) {
      std::uniform_int_distribution<int> dist(0, i);
      const int j = dist(gen);
      if (j < P.max_num_best_mappings) sel[j] = i;
    }
    std::sort(sel.begin(), sel.end());
  }
  int idx = 0, reported = 0;
  const int to_report = std::min(P.max_num_best_mappings, ps.n_best);
  const uint8_t uniq = (ps.n_best == 1 || rs[0].n_best == 1 || rs[1].n_best == 1) ? 1 : 0;
  static const int DIR_S1[4] = {0, 1, 0, 1}, DIR_S2[4] = {1, 0, 0, 1};
  const int n_dirs = P.split_alignment ? 4 : 2;
  for (int dir = 0; dir < n_dirs && reported != to_report; ++dir) {  // mapping_generator.h:486-654
    const int s1 = DIR_S1[dir], s2 = DIR_S2[dir];
    const std::vector<Draft> &m1 = rs[0].map[s1], &m2 = rs[1].map[s2];
    for (const auto &bp : ps.best[dir]) {
      const Draft &d1 = m1[bp.first], &d2 = m2[bp.second];
      if (d1.err + d2.err > ps.min_sum) continue;
      if (idx == sel[reported]) {
        u32 st1, en1, st2, en2;
        uint8_t q;
        if (P.split_alignment) {
          ref_span_split(P, ref, d1, s1, rs[0].split[s1][bp.first], s1 == 0 ? r[0].data() : neg[0].data(), L[0], st1, en1);
          ref_span_split(P, ref, d2, s2, rs[1].split[s2][bp.second], s2 == 0 ? r[1].data() : neg[1].data(), L[1], st2, en2);
          const uint16_t al1 = en1 - st1 + 1, al2 = en2 - st2 + 1;
          uint8_t q1 = mapq_se_split(P, s1, d1.err, al1, L[0], 2, rs[0]);
          uint8_t q2 = mapq_se_split(P, s2, d2.err, al2, L[1], 2, rs[1]);
          q1 *= 1.2; if (q1 > 60) q1 = 60;   // mapping_generator.h:1171-1179 (no mate mixing under split alignment)
          q2 *= 1.2; if (q2 > 60) q2 = 60;
          q = q1 < q2 ? q1 : q2;
          if (q < 60 && force >= 0 && force < q) q = force;
          if (reported < cap) {  // mapping_generator.cc:169-210
            orc_pairs_record &o = reinterpret_cast<orc_pairs_record *>(out)[reported];
            int rid1 = (u32)(d1.pos >> 32), rid2 = (u32)(d2.pos >> 32);
            int pos1 = s1 == 0 ? st1 : en1, pos2 = s2 == 0 ? st2 : en2;
            uint8_t str1 = s1 == 0 ? 1 : 0, str2 = s2 == 0 ? 1 : 0;
            const bool smaller = rid1 < rid2 || (rid1 == rid2 && pos1 < pos2);  // identity chromosome ranks
            if (!smaller) { std::swap(rid1, rid2); std::swap(pos1, pos2); std::swap(str1, str2); }
            o.read_id = read_id; o.rid1 = rid1; o.rid2 = rid2; o.pos1 = pos1; o.pos2 = pos2;
            o.strand1 = str1; o.strand2 = str2; o.mapq = q; o.is_unique = uniq;
          }
          if (++reported == to_report) break;
          ++idx;
          continue;
        }
        if (sam && sam->paf) {  // PairedPAFMapping: BED-branch spans, per-mate MAPQs
          ref_span(P, ref, d1, s1 == 0 ? r[0].data() : neg[0].data(), L[0], st1, en1);
          ref_span(P, ref, d2, s2 == 0 ? r[1].data() : neg[1].data(), L[1], st2, en2);
          const uint16_t pal1 = en1 - st1 + 1, pal2 = en2 - st2 + 1;
          PafRec o;
          o.mapq = mapq_pe(d1.err, d2.err, pal1, pal2, L[0], L[1], force, ps, rs);
          o.mapq1 = o.mapq2 = o.mapq;  // mapping_generator.h:611-612: both mates' mapq fields are overwritten with the pair's before the record is built
          const uint16_t frag = (uint16_t)(s1 == 0 ? (int)(en2 - st1 + 1) : (int)(en1 - st2 + 1));
          const uint16_t pos_al = s1 == 0 ? pal1 : pal2, neg_al = s1 == 1 ? pal1 : pal2;
          o.read_id = read_id; o.rid = (u32)(d1.pos >> 32); o.start = s1 == 0 ? st1 : st2; o.name1 = sam->name1; o.name2 = sam->name2;
          o.len1 = (uint16_t)L[0]; o.len2 = (uint16_t)L[1];
          o.frag = neg_al; o.pal = frag; o.nal = pos_al;  // the argument order quirk, see PafRec
          o.dir = s1 == 0 ? 1 : 0; o.uniq = uniq; o.dups = 1;
          sam->paf->push_back(o);
          if (++reported == to_report) break;
          ++idx;
          continue;
        }
        if (sam) {  // mapping_generator.h:575-640 with MAPPINGFORMAT_SAM, mapping_generator.cc:84-107
          SamRec a, b;
          ref_span_sam(P, ref, d1, s1 == 0 ? r[0].data() : neg[0].data(), L[0], st1, en1, a);
          ref_span_sam(P, ref, d2, s2 == 0 ? r[1].data() : neg[1].data(), L[1], st2, en2, b);
          const uint16_t sal1 = en1 - st1 + 1, sal2 = en2 - st2 + 1;
          q = mapq_pe(d1.err, d2.err, sal1, sal2, L[0], L[1], force, ps, rs);
          const int tlen = s1 == 0 ? (int)(en2 - st1 + 1) : (int)(en1 - st2 + 1);
          int f1 = 3 | 64, f2 = 3 | 128;
          if (s1 == 1) { f1 |= 16; f2 |= 32; }
          if (s2 == 1) { f1 |= 32; f2 |= 16; }
          if (reported >= 1) { f1 |= 256; f2 |= 256; }
          a.read_id = b.read_id = read_id; a.name = sam->name1; b.name = sam->name2;
          a.pos = st1; a.rid = (int)(u32)(d1.pos >> 32); b.pos = st2; b.rid = (int)(u32)(d2.pos >> 32);
          a.mpos = b.pos; a.mrid = b.rid; b.mpos = a.pos; b.mrid = a.rid;
          a.strand_pos = s1 == 0; b.strand_pos = s2 == 0;
          a.tlen = a.strand_pos ? tlen : -tlen; b.tlen = b.strand_pos ? tlen : -tlen;
          a.flag = f1; b.flag = f2; a.is_unique = b.is_unique = uniq; a.mapq = b.mapq = q;
          a.seq = s1 == 0 ? r[0] : neg[0]; b.seq = s2 == 0 ? r[1] : neg[1];
          a.qual = sam->qual1; b.qual = sam->qual2;
          if (s1 != 0) std::reverse(a.qual.begin(), a.qual.end());
          if (s2 != 0) std::reverse(b.qual.begin(), b.qual.end());
          a.qual.resize(a.seq.size(), 'I'); b.qual.resize(b.seq.size(), 'I');
          sam->recs->push_back(a); sam->recs->push_back(b);
          if (++reported == to_report) break;
          ++idx;
          continue;
        }
        ref_span(P, ref, d1, s1 == 0 ? r[0].data() : neg[0].data(), L[0], st1, en1);
        ref_span(P, ref, d2, s2 == 0 ? r[1].data() : neg[1].data(), L[1], st2, en2);
        const uint16_t al1 = en1 - st1 + 1, al2 = en2 - st2 + 1;
        q = mapq_pe(d1.err, d2.err, al1, al2, L[0], L[1], force, ps, rs);
        if (reported < cap) {
          orc_pe_record &o = out[reported];
          o.read_id = read_id;
          o.rid = (u32)(d1.pos >> 32);
          o.fragment_start = s1 == 0 ? st1 : st2;
          o.fragment_length = (uint16_t)(s1 == 0 ? (int)(en2 - st1 + 1) : (int)(en1 - st2 + 1));
          o.mapq = q;
          o.direction = s1 == 0 ? 1 : 0;
          o.is_unique = uniq;
          o.num_dups = 1;
          o.positive_alignment_length = s1 == 0 ? al1 : al2;
          o.negative_alignment_length = s1 == 1 ? al1 : al2;
        }
        if (++reported == to_report) break;
      }
      ++idx;
    }
  }
  if (tr) tr->n_records = reported;
  return reported;
}

static int map_one_pair(const orc_params &P, const orc_index &ix, const orc_reference &ref, std::mt19937 &gen,
                        const char *s1, u32 len1, const char *s2, u32 len2, u32 read_id, u32 pair_index,
                        orc_pe_record *out, int cap, orc_pair_trace *tr, const SamSink *sam = nullptr) {
  if (tr) memset(tr, 0, sizeof(*tr));
  if (len1 < (u32)P.min_read_length || len2 < (u32)P.min_read_length) return 0;
  std::string r[2] = {std::string(s1, len1), std::string(s2, len2)}, neg[2];
  revcomp(r[0].data(), len1, neg[0]);
  revcomp(r[1].data(), len2, neg[1]);
  if (P.trim_adapters) trim_adapters(P, r[0], r[1], neg[0], neg[1]);
  const u32 L[2] = {(u32)r[0].size(), (u32)r[1].size()};
  if (tr) { tr->trimmed_len[0] = L[0]; tr->trimmed_len[1] = L[1]; }
  ReadState rs[2];
  rs[0].reset(); rs[1].reset();
  gen_minimizers(r[0].data(), L[0], pair_index, ix.k, ix.w, rs[0].mm);
  gen_minimizers(r[1].data(), L[1], pair_index, ix.k, ix.w, rs[1].mm);
  if (tr) { tr->n_minimizers[0] = rs[0].mm.size(); tr->n_minimizers[1] = rs[1].mm.size(); }
  if (rs[0].mm.empty() || rs[1].mm.empty()) return 0;
  gen_candidates(P, ix, rs[0]);
  gen_candidates(P, ix, rs[1]);
  if (tr) for (int m = 0; m < 2; ++m) { tr->n_pos_candidates_gen[m] = rs[m].cand[0].size(); tr->n_neg_candidates_gen[m] = rs[m].cand[1].size(); }
  int sup = 0;
  if (!P.split_alignment) sup = supplement(P, ix, rs);
  if (tr) tr->supplement_result = sup;
  size_t nc1 = rs[0].cand[0].size() + rs[0].cand[1].size(), nc2 = rs[1].cand[0].size() + rs[1].cand[1].size();
  if (nc1 > 0 && nc2 > 0 && !P.split_alignment) {
    for (int m = 0; m < 2; ++m) for (int s = 0; s < 2; ++s) { rs[m].cand[s].swap(rs[m].buf[s]); rs[m].cand[s].clear(); }
    pe_filter_dir(P.max_insert_size, rs[0].buf[0], rs[1].buf[1], rs[0].cand[0], rs[1].cand[1]);
    pe_filter_dir(P.max_insert_size, rs[0].buf[1], rs[1].buf[0], rs[0].cand[1], rs[1].cand[0]);
    nc1 = rs[0].cand[0].size() + rs[0].cand[1].size();
    nc2 = rs[1].cand[0].size() + rs[1].cand[1].size();
  }
  if (tr) for (int m = 0; m < 2; ++m) {
    tr->n_pos_candidates[m] = rs[m].cand[0].size(); tr->n_neg_candidates[m] = rs[m].cand[1].size();
    tr->repetitive_seed_length[m] = rs[m].rep_len;
  }
  if (!(nc1 > 0 && nc2 > 0)) return 0;
  if (P.split_alignment) {
    verify_read_split(P, ref, r[0].data(), neg[0], L[0], rs[0]);
    verify_read_split(P, ref, r[1].data(), neg[1], L[1], rs[1]);
  } else {
    verify_read(P, ref, r[0].data(), neg[0], L[0], rs[0]);
    verify_read(P, ref, r[1].data(), neg[1], L[1], rs[1]);
  }
  if (tr) for (int m = 0; m < 2; ++m) {
    tr->n_pos_mappings[m] = rs[m].map[0].size(); tr->n_neg_mappings[m] = rs[m].map[1].size();
    tr->min_errors[m] = rs[m].min_err; tr->second_min_errors[m] = rs[m].second_min_err;
    tr->n_best[m] = rs[m].n_best; tr->n_second_best[m] = rs[m].n_second_best;
  }
  return finish_pair(P, ref, gen, r, neg, L, rs, sup, read_id, out, cap, tr, sam);
}

// Single-end: the taskloop body of MapSingleEndReads (chromap.h:383-470) + GenerateBestMappingsForSingleEndRead /
// ProcessBestMappingsForSingleEndRead (mapping_generator.h:115-157,256-343) + EmplaceBackSingleEndMappingRecord
// (mapping_generator.cc:7-16).  No mate: no supplementation, no paired-end filter, mappings stay in verification
// order; the sampling generator is a fresh mt19937(11) per read (mapping_generator.h:128).
static int map_one_read_se(const orc_params &P, const orc_index &ix, const orc_reference &ref, const char *s, u32 len, u32 read_id,
                           u32 read_index, orc_pe_record *out, int cap, const SamSink *sam = nullptr) {
  if (len < (u32)P.min_read_length) return 0;
  std::string r(s, len), neg;
  revcomp(r.data(), len, neg);
  ReadState rs;
  rs.reset();
  gen_minimizers(r.data(), len, read_index, ix.k, ix.w, rs.mm);
  if (rs.mm.empty()) return 0;
  gen_candidates(P, ix, rs);
  if (rs.cand[0].size() + rs.cand[1].size() == 0) return 0;
  verify_read(P, ref, r.data(), neg, len, rs);
  if (rs.map[0].size() + rs.map[1].size() == 0) return 0;
  std::vector<int> sel(P.max_num_best_mappings);
  std::iota(sel.begin(), sel.end(), 0);
  if (rs.n_best > P.max_num_best_mappings) {
    std::mt19937 gen(11);
    for (int i = P.max_num_best_mappings; i < rs.n_best; ++i) {
      std::uniform_int_distribution<int> dist(0, i);
      const int j = dist(gen);
      if (j < P.max_num_best_mappings) sel[j] = i;
    }
    std::sort(sel.begin(), sel.end());
  }
  int idx = 0, reported = 0;
  const int to_report = std::min(rs.n_best, P.max_num_best_mappings);
  for (int st = 0; st < 2 && reported != to_report; ++st) {
    for (const Draft &d : rs.map[st]) {
      if (d.err > rs.min_err) continue;
      if (idx == sel[reported]) {
        u32 a, b;
        if (sam && sam->paf) {  // PAFMapping (mapping_generator.cc:31-41)
          ref_span(P, ref, d, st == 0 ? r.data() : neg.data(), len, a, b);
          const uint16_t al = b - a + 1;
          PafRec o;
          o.read_id = read_id; o.rid = (u32)(d.pos >> 32); o.start = a; o.name1 = sam->name1; o.len1 = (uint16_t)len; o.len2 = 0;
          o.frag = al; o.pal = o.nal = 0; o.mapq = mapq_se(d.err, al, (int)len, P.error_threshold, rs); o.mapq1 = o.mapq2 = 0;
          o.dir = st == 0 ? 1 : 0; o.uniq = rs.n_best == 1 ? 1 : 0; o.dups = 1;
          sam->paf->push_back(o);
          if (++reported == to_report) break;
          ++idx;
          continue;
        }
        if (sam) {  // mapping_generator.h:302-331 with MAPPINGFORMAT_SAM
          SamRec sr;
          ref_span_sam(P, ref, d, st == 0 ? r.data() : neg.data(), len, a, b, sr);
          const uint16_t al = b - a + 1;
          sr.read_id = read_id; sr.name = sam->name1; sr.pos = a; sr.rid = (int)(u32)(d.pos >> 32); sr.mpos = 0; sr.mrid = -1; sr.tlen = 0;
          sr.flag = (st == 0 ? 0 : 16) | (reported >= 1 ? 256 : 0);
          sr.strand_pos = st == 0; sr.is_unique = rs.n_best == 1; sr.mapq = mapq_se(d.err, al, (int)len, P.error_threshold, rs);
          sr.seq = st == 0 ? r : neg;
          sr.qual = sam->qual1;
          if (st != 0) std::reverse(sr.qual.begin(), sr.qual.end());
          sam->recs->push_back(sr);
          if (++reported == to_report) break;
          ++idx;
          continue;
        }
        ref_span(P, ref, d, st == 0 ? r.data() : neg.data(), len, a, b);
        const uint16_t al = b - a + 1;
        if (reported < cap) {
          orc_pe_record &o = out[reported];
          memset(&o, 0, sizeof(o));
          o.read_id = read_id; o.rid = (u32)(d.pos >> 32); o.fragment_start = a; o.fragment_length = al;
          o.mapq = mapq_se(d.err, al, (int)len, P.error_threshold, rs);
          o.direction = st == 0 ? 1 : 0; o.is_unique = rs.n_best == 1 ? 1 : 0; o.num_dups = 1;
        }
        if (++reported == to_report) break;
      }
      ++idx;
    }
  }
  return reported;
}

// ----------------------------------------------------------------------------------------------
// Host-side pieces: FASTA/FASTQ reader (kseq.h semantics: name = first token, multi-line sequence),
// index file I/O, post-processing, BED text.
struct SeqReader {
  gzFile f = nullptr;
  std::vector<char> buf;
  size_t pos = 0, end = 0;
  int last = 0;  // pending header char
  bool eof = false;
  bool open(const char *p) { f = gzopen(p, "r"); buf.resize(1 << 20); return f != nullptr; }
  void close() { if (f) gzclose(f); f = nullptr; }
  int getc_() {
    if (pos >= end) {
      if (eof) return -1;
      int n = gzread(f, buf.data(), buf.size());
      if (n <= 0) { eof = true; return -1; }
      pos = 0; end = n;
    }
    return (unsigned char)buf[pos++];
  }
  bool getline_(std::string &s) {  // without the newline; false at EOF with nothing read
    s.clear();
    int c;
    bool any = false;
    while ((c = getc_()) != -1) {
      any = true;
      if (c == '\n') break;
      s.push_back((char)c);
    }
    if (!s.empty() && s.back() == '\r') s.pop_back();
    return any;
  }
  // returns false at EOF
  bool next(std::string &name, std::string &seq, std::string &qual) {
    name.clear(); seq.clear(); qual.clear();
    int c;
    if (last == 0) {
      while ((c = getc_()) != -1 && c != '>' && c != '@') {}
      if (c == -1) return false;
      last = c;
    }
    std::string line;
    getline_(line);
    size_t sp = line.find_first_of(" \t");
    name = sp == std::string::npos ? line : line.substr(0, sp);
    last = 0;
    while ((c = getc_()) != -1 && c != '>' && c != '+' && c != '@') {
      if (c == '\n') continue;
      seq.push_back((char)c);
      std::string rest;
      getline_(rest);
      seq += rest;
    }
    if (c == '>' || c == '@') last = c;
    if (c != '+') return true;
    getline_(line);  // rest of '+' line
    while (qual.size() < seq.size()) {
      std::string q;
      if (!getline_(q)) break;
      qual += q;
    }
    return true;
  }
};

extern "C" {

void orc_default_params(orc_params *p) {
  p->error_threshold = 8; p->min_num_seeds = 2; p->max_seed_freq0 = 500; p->max_seed_freq1 = 1000;
  p->max_num_best_mappings = 1; p->max_insert_size = 1000; p->mapq_threshold = 30; p->min_read_length = 30;
  p->drop_repetitive_reads = 500000; p->trim_adapters = 0; p->remove_pcr_duplicates = 0; p->tn5_shift = 0;
  p->split_alignment = 0; p->low_memory_mode = 0; p->output_format = 1;
  p->single_end = 0;
}

int orc_apply_preset(orc_params *p, const char *preset) {  // chromap_driver.cc:247-275
  std::string s = preset ? preset : "";
  if (s.empty()) return 0;
  if (s == "atac") { p->max_insert_size = 2000; p->trim_adapters = 1; p->remove_pcr_duplicates = 1; p->tn5_shift = 1; p->low_memory_mode = 1; p->output_format = 1; return 0; }
  if (s == "chip") { p->max_insert_size = 2000; p->remove_pcr_duplicates = 1; p->low_memory_mode = 1; p->output_format = 1; return 0; }
  if (s == "hic") { p->error_threshold = 4; p->mapq_threshold = 1; p->split_alignment = 1; p->low_memory_mode = 1; p->output_format = 5; return 0; }
  return -1;
}

orc_reference *orc_reference_load(const char *path) {
  SeqReader rd;
  if (!rd.open(path)) return nullptr;
  orc_reference *r = new orc_reference;
  std::string n, s, q;
  while (rd.next(n, s, q)) {
    if (s.empty()) continue;  // sequence_batch.cc:84-118 keeps only length > 0
    r->names.push_back(n);
    r->lens.push_back(s.size());
    s.append(64, '\0');
    r->seqs.push_back(std::move(s));
  }
  rd.close();
  return r;
}
orc_reference *orc_reference_from_memory(uint32_t n, const char *concat, const uint64_t *off, const char *const *names) {
  orc_reference *r = new orc_reference;
  for (u32 i = 0; i < n; ++i) {
    std::string s(concat + off[i], off[i + 1] - off[i]);
    r->lens.push_back(s.size());
    s.append(64, '\0');
    r->seqs.push_back(std::move(s));
    r->names.push_back(names ? names[i] : ("chr" + std::to_string(i + 1)));
  }
  return r;
}
void orc_reference_free(orc_reference *r) { delete r; }
uint32_t orc_reference_num_sequences(const orc_reference *r) { return r->seqs.size(); }
uint32_t orc_reference_length(const orc_reference *r, uint32_t rid) { return r->lens[rid]; }
const char *orc_reference_name(const orc_reference *r, uint32_t rid) { return r->names[rid].c_str(); }
const char *orc_reference_seq(const orc_reference *r, uint32_t rid) { return r->seqs[rid].data(); }

orc_index *orc_index_load(const char *path) {  // index.cc:132-169, khash.h:358-373
  FILE *f = fopen(path, "rb");
  if (!f) return nullptr;
  orc_index *ix = new orc_index;
  u32 lookup_size = 0, n_occ = 0;
  bool ok = fread(&ix->k, 4, 1, f) == 1 && fread(&ix->w, 4, 1, f) == 1 && fread(&lookup_size, 4, 1, f) == 1;
  ok = ok && fread(&ix->n_buckets, 4, 1, f) == 1 && fread(&ix->size, 4, 1, f) == 1 &&
       fread(&ix->n_occupied, 4, 1, f) == 1 && fread(&ix->upper_bound, 4, 1, f) == 1;
  if (ok && ix->n_buckets) {
    const size_t fs = ix->n_buckets < 16 ? 1 : ix->n_buckets >> 4;
    ix->flags.resize(fs); ix->keys.resize(ix->n_buckets); ix->vals.resize(ix->n_buckets);
    ok = fread(ix->flags.data(), 4, fs, f) == fs && fread(ix->keys.data(), 8, ix->n_buckets, f) == ix->n_buckets &&
         fread(ix->vals.data(), 8, ix->n_buckets, f) == ix->n_buckets;
  }
  ok = ok && fread(&n_occ, 4, 1, f) == 1;
  if (ok && n_occ) { ix->occ.resize(n_occ); ok = fread(ix->occ.data(), 8, n_occ, f) == n_occ; }
  fclose(f);
  if (!ok) { delete ix; return nullptr; }
  return ix;
}

int orc_index_save(const orc_index *ix, const char *path) {  // index.cc:91-130, khash.h:374-386
  FILE *f = fopen(path, "wb");
  if (!f) return -1;
  fwrite(&ix->k, 4, 1, f); fwrite(&ix->w, 4, 1, f); fwrite(&ix->size, 4, 1, f);
  fwrite(&ix->n_buckets, 4, 1, f); fwrite(&ix->size, 4, 1, f); fwrite(&ix->n_occupied, 4, 1, f); fwrite(&ix->upper_bound, 4, 1, f);
  if (ix->n_buckets) {
    fwrite(ix->flags.data(), 4, ix->flags.size(), f);
    fwrite(ix->keys.data(), 8, ix->n_buckets, f);
    fwrite(ix->vals.data(), 8, ix->n_buckets, f);
  }
  const u32 n_occ = ix->occ.size();
  fwrite(&n_occ, 4, 1, f);
  if (n_occ) fwrite(ix->occ.data(), 8, n_occ, f);
  fclose(f);
  return 0;
}

orc_index *orc_index_build(const orc_reference *ref, int k, int w) {  // index.cc:12-89
  std::vector<Mm> all;
  for (u32 i = 0; i < ref->seqs.size(); ++i) gen_minimizers(ref->seqs[i].data(), ref->lens[i], i, k, w, all);
  std::stable_sort(all.begin(), all.end(), [](const Mm &a, const Mm &b) { return a.hash < b.hash || (a.hash == b.hash && a.hit < b.hit); });
  orc_index *ix = new orc_index;
  ix->k = k; ix->w = w;
  size_t n_keys = 0;
  for (size_t i = 0; i < all.size(); ++i) if (i == 0 || all[i].hash != all[i - 1].hash) ++n_keys;
  u32 nb = 4;
  while ((u32)(nb * 0.77 + 0.5) < n_keys) nb <<= 1;  // kh_put grows when n_occupied >= upper_bound
  ix->n_buckets = nb; ix->size = ix->n_occupied = n_keys; ix->upper_bound = (u32)(nb * 0.77 + 0.5);
  ix->flags.assign(nb < 16 ? 1 : nb >> 4, 0xaaaaaaaau);
  ix->keys.assign(nb, 0); ix->vals.assign(nb, 0);
  const u32 m = nb - 1;
  for (size_t i = 0; i < all.size();) {
    size_t j = i;
    while (j < all.size() && all[j].hash == all[i].hash) ++j;
    u64 key = all[i].hash << 1, val;
    if (j - i == 1) { key |= 1; val = all[i].hit; }
    else { val = ((u64)ix->occ.size() << 32) | (u32)(j - i); for (size_t t = i; t < j; ++t) ix->occ.push_back(all[t].hit); }
    u32 b = (u32)(all[i].hash) & m, step = 0;
    while (!((ix->flags[b >> 4] >> ((b & 0xfU) << 1)) & 2)) b = (b + (++step)) & m;
    ix->flags[b >> 4] &= ~(3u << ((b & 0xfU) << 1));
    ix->keys[b] = key; ix->vals[b] = val;
    i = j;
  }
  return ix;
}
orc_index *orc_index_from_arrays(int k, int w, uint32_t n_buckets, const uint32_t *flags, const uint64_t *keys,
                                  const uint64_t *vals, const uint64_t *occ, uint32_t n_occ) {
  orc_index *ix = new orc_index;
  ix->k = k; ix->w = w; ix->n_buckets = n_buckets;
  const size_t nf = n_buckets < 16 ? 1 : n_buckets >> 4;
  ix->flags.assign(flags, flags + nf);
  ix->keys.assign(keys, keys + n_buckets);
  ix->vals.assign(vals, vals + n_buckets);
  ix->occ.assign(occ, occ + n_occ);
  u32 sz = 0;
  for (u32 i = 0; i < n_buckets; ++i) if (((ix->flags[i >> 4] >> ((i & 0xfU) << 1)) & 3) == 0) ++sz;
  ix->size = ix->n_occupied = sz;
  ix->upper_bound = (u32)(n_buckets * 0.77 + 0.5);
  return ix;
}
void orc_index_free(orc_index *ix) { delete ix; }
int orc_index_k(const orc_index *ix) { return ix->k; }
int orc_index_w(const orc_index *ix) { return ix->w; }
uint32_t orc_index_arrays(const orc_index *ix, const uint32_t **flags, const uint64_t **keys, const uint64_t **vals,
                          const uint64_t **occ, uint32_t *n_occ) {
  *flags = ix->flags.data(); *keys = ix->keys.data(); *vals = ix->vals.data(); *occ = ix->occ.data(); *n_occ = ix->occ.size();
  return ix->n_buckets;
}
int orc_index_lookup(const orc_index *ix, uint64_t h, uint64_t *key, uint64_t *val) {
  u64 k, v;
  if (!ix->lookup(h, k, v)) return 0;
  *key = k; *val = v;
  return 1;
}

int orc_minimizers(const char *seq, uint32_t len, uint32_t seq_index, int k, int w, uint64_t *hash, uint64_t *hit, int cap) {
  std::vector<Mm> v;
  gen_minimizers(seq, len, seq_index, k, w, v);
  for (size_t i = 0; i < v.size() && (int)i < cap; ++i) { hash[i] = v[i].hash; hit[i] = v[i].hit; }
  return v.size();
}
int orc_banded_align(int e, const char *pattern, const char *text, int read_len, int *end_pos) { return banded_align(e, pattern, text, read_len, end_pos); }
void orc_banded_traceback(int e, int min_errors, const char *pattern, const char *text, int read_len, int *start_pos) { banded_traceback(e, min_errors, pattern, text, read_len, start_pos); }
int orc_adjust_gap_beginning(int strand, const char *ref, const char *read, int *gap, int read_end, int ref_start, int ref_end) {
  return adjust_gap_beginning(strand, ref, read, gap, read_end, ref_start, ref_end);
}
// the mate-guided lookup (index.cc:351-489) over records that were probed elsewhere, for tests of the device formulations:
// kind[i] 0 absent / 1 singleton / 2 multi, val[i] the table value, mm_hit[i] = read position << 1 | strand
int orc_rescue_test(int k, int w, int max_seed_freq0, int min_num_seeds, int strand, uint32_t range, int n_mm, const uint8_t *kind,
                    const uint64_t *val, const uint64_t *mm_hit, const uint64_t *occ, const uint64_t *mate_pos, const uint8_t *mate_cnt,
                    int n_mate, uint32_t *rep_len, uint64_t *hits, int cap, int *nh) {
  std::vector<Cand> mate((size_t)n_mate);
  for (int i = 0; i < n_mate; ++i) { mate[i].pos = mate_pos[i]; mate[i].cnt = mate_cnt[i]; }
  std::vector<u64> out;
  u32 rl = 0;
  const int r = rescue_core(k, w, max_seed_freq0, min_num_seeds, strand, range, (size_t)n_mm,
                            [&](size_t i, u64 &key, u64 &v, u64 &mhit) { mhit = mm_hit[i]; v = val[i]; key = kind[i] == 1 ? 1 : 0; return kind[i] != 0; },
                            occ, mate, rl, out);
  *rep_len = rl;
  *nh = (int)out.size();
  for (size_t i = 0; i < out.size() && (int)i < cap; ++i) hits[i] = out[i];
  return r;
}
// GenerateDraftMappings (non-split, draft_mapping_generator.cc:9-357) for one read over given candidate lists, for tests of
// the device formulations.  ref: one sequence of ref_len bases (followed by >= 64 NUL); cand_pos / cand_cnt: [2][n_cand[s]]
// laid out strand after strand; out_pos / out_err: [2][cap].  stats: min_err, n_best, second_min_err, n_second_best.
void orc_verify_test(int e, const char *ref_seq, uint32_t ref_len, const char *read, uint32_t L, int n_mm, const int *n_cand,
                     const uint64_t *cand_pos, const uint8_t *cand_cnt, int cap, int *n_map, uint64_t *out_pos, int16_t *out_err, int *stats) {
  orc_params P;
  orc_default_params(&P);
  P.error_threshold = e;
  orc_reference ref;
  ref.names.push_back("t");
  ref.lens.push_back(ref_len);
  std::string sq(ref_seq, ref_len);
  sq.append(64, '\0');
  ref.seqs.push_back(std::move(sq));
  ReadState rs;
  rs.reset();
  rs.mm.resize((size_t)n_mm);
  size_t o = 0;
  for (int s = 0; s < 2; ++s)
    for (int i = 0; i < n_cand[s]; ++i, ++o) { Cand c; c.pos = cand_pos[o]; c.cnt = cand_cnt[o]; rs.cand[s].push_back(c); }
  std::string neg;
  revcomp(read, L, neg);
  verify_read(P, ref, read, neg, L, rs);
  for (int s = 0; s < 2; ++s) {
    n_map[s] = (int)rs.map[s].size();
    for (size_t i = 0; i < rs.map[s].size() && (int)i < cap; ++i) { out_pos[(size_t)s * cap + i] = rs.map[s][i].pos; out_err[(size_t)s * cap + i] = (int16_t)rs.map[s][i].err; }
  }
  stats[0] = rs.min_err; stats[1] = rs.n_best; stats[2] = rs.second_min_err; stats[3] = rs.n_second_best;
}
// best-pair statistics of one read pair (mapping_generator.h:160-197 + :346-484, non-split) over given draft mappings, for
// tests of the device formulations.  n_map: {mate 1 +, mate 1 -, mate 2 +, mate 2 -}; pos / err: the four lists one after the
// other, in any order (SortMappingsByPositions is applied here).  stats: min_sum, n_best, second_min_sum, n_second_best.
void orc_pair_stats_test(int e, int max_insert_size, int min_read_length, uint32_t L1, uint32_t L2, const int *n_map, const uint64_t *pos,
                         const int16_t *err, int *stats) {
  orc_params P;
  orc_default_params(&P);
  P.error_threshold = e; P.max_insert_size = max_insert_size; P.min_read_length = min_read_length;
  std::vector<Draft> m[4];
  size_t o = 0;
  for (int q = 0; q < 4; ++q)
    for (int i = 0; i < n_map[q]; ++i, ++o) m[q].push_back({(int)err[o], pos[o]});
  auto by_pos = [](const Draft &a, const Draft &b) { return a.pos != b.pos ? a.pos < b.pos : a.err < b.err; };
  for (int q = 0; q < 4; ++q) std::sort(m[q].begin(), m[q].end(), by_pos);
  PairState ps;
  ps.min_sum = 2 * e + 1; ps.n_best = 0; ps.second_min_sum = ps.min_sum; ps.n_second_best = 0;
  pair_dir(P, 0, L1, L2, m[0], m[3], ps, ps.best[0]);
  pair_dir(P, 1, L1, L2, m[1], m[2], ps, ps.best[1]);
  stats[0] = ps.min_sum; stats[1] = ps.n_best; stats[2] = ps.second_min_sum; stats[3] = ps.n_second_best;
}
// The part of the taskloop body after verification (SortMappingsByPositions, best pairs, sampling with a fresh
// std::mt19937(11), spans, MAPQ, BED records) for one pair over given draft mappings, for tests of the device emit kernels.
// n_map / pos / err as in orc_pair_stats_test; tally: {min_err, n_best, second_min_err, n_second_best} of mate 1 then mate 2.
int orc_emit_test(const orc_params *p, const char *ref_seq, uint32_t ref_len, const char *read1, uint32_t L1, const char *read2, uint32_t L2,
                  const int *n_map, const uint64_t *pos, const int16_t *err, const int *tally, const uint32_t *rep_len, int sup, uint32_t read_id,
                  orc_pe_record *out, int cap) {
  orc_reference ref;
  ref.names.push_back("t");
  ref.lens.push_back(ref_len);
  std::string sq(ref_seq, ref_len);
  sq.append(64, '\0');
  ref.seqs.push_back(std::move(sq));
  const std::string r[2] = {std::string(read1, L1), std::string(read2, L2)};
  std::string neg[2];
  revcomp(r[0].data(), L1, neg[0]);
  revcomp(r[1].data(), L2, neg[1]);
  const u32 L[2] = {L1, L2};
  ReadState rs[2];
  size_t o = 0;
  for (int m = 0; m < 2; ++m) {
    rs[m].reset();
    for (int st = 0; st < 2; ++st)
      for (int i = 0; i < n_map[2 * m + st]; ++i, ++o) rs[m].map[st].push_back({(int)err[o], pos[o]});
    rs[m].min_err = tally[4 * m]; rs[m].n_best = tally[4 * m + 1]; rs[m].second_min_err = tally[4 * m + 2]; rs[m].n_second_best = tally[4 * m + 3];
    rs[m].rep_len = rep_len[m];
  }
  std::mt19937 gen(11);
  return finish_pair(*p, ref, gen, r, neg, L, rs, sup, read_id, out, cap, nullptr, nullptr);
}
// CorrectBarcodeAt (chromap.cc:572-799) for one barcode, for tests of the device kernel: returns 1 if the (possibly corrected)
// barcode is in the whitelist; *out_key = the 2-bit key of the barcode afterwards; counters as the mapper keeps them.
int orc_correct_barcode_test(const orc_whitelist *wl, int err_threshold, double prob_threshold, const char *bc, const char *qual, uint32_t len,
                             uint64_t *out_key, uint64_t *n_in_whitelist, uint64_t *n_corrected) {
  std::string b(bc, len);
  const bool ok = correct_barcode(*wl, err_threshold, prob_threshold, &b[0], qual, len, n_in_whitelist, n_corrected);
  *out_key = barcode_seed(b.data(), len);
  return ok ? 1 : 0;
}
// the two drop-off aligners of the split path (alignment.cc:197-283 / :285-376), for tests of the device formulation
int orc_align_dropoff(int e, const char *pattern, const char *text, int read_len, int from_3_end, int *end_pos, int *read_len_out) {
  return from_3_end ? align_dropoff_3end(e, pattern, text, read_len, end_pos, read_len_out) : align_dropoff(e, pattern, text, read_len, end_pos, read_len_out);
}

orc_mapper *orc_mapper_create(const orc_params *p, const orc_index *ix, const orc_reference *ref) {
  if (p->error_threshold >= 16) return nullptr;
  if (!((p->output_format == 1 && !p->split_alignment) || (p->output_format == 5 && p->split_alignment))) return nullptr;  // BED or Hi-C pairs
  orc_mapper *m = new orc_mapper;
  m->P = *p; m->ix = ix; m->ref = ref;
  return m;
}
void orc_mapper_free(orc_mapper *m) { delete m; }

extern "C" int64_t orc_map_pairs_mt(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2,
                         const uint32_t *off2, uint32_t first_read_id, orc_pe_record *out, int64_t cap_out, int n_threads,
                         orc_pair_trace *trace);
// Chunking of `#pragma omp taskloop grainsize(5000)` (chromap.h:892) by this image's libgomp (measured with
// a stand-alone OpenMP probe): num_tasks = n/5000 (min 1); chunk = n/num_tasks, the first n%num_tasks
// chunks one longer.  `generator` (chromap.h:863) is private to the parallel region, hence FIRSTPRIVATE
// in every generated task: each chunk starts from a fresh copy of mt19937(11) and only pairs inside the
// same chunk share a sampling stream.  So multi-mapper choices depend on (pair index in batch, batch
// size) only — not on the thread count or the order tasks run in.
int orc_ref_task_chunks(uint32_t n, uint32_t *starts, uint32_t *ends, int cap) {
  u32 nt = n / 5000;
  if (nt < 1) nt = 1;
  if ((int)nt > cap) return -1;
  const u32 chunk = n / nt, rem = n % nt;
  u32 s = 0;
  for (u32 t = 0; t < nt; ++t) { const u32 len = chunk + (t < rem ? 1 : 0); starts[t] = s; ends[t] = s + len; s += len; }
  return nt;
}

int64_t orc_map_pairs(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2,
                      const uint32_t *off2, uint32_t first_read_id, orc_pe_record *out, int64_t cap_out,
                      orc_pair_trace *trace) {
  return orc_map_pairs_mt(m, n, seq1, off1, seq2, off2, first_read_id, out, cap_out, 1, trace);
}

int64_t orc_map_pairs_mt(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2,
                         const uint32_t *off2, uint32_t first_read_id, orc_pe_record *out, int64_t cap_out, int n_threads,
                         orc_pair_trace *trace) {
  const int per = m->P.max_num_best_mappings;
  std::vector<orc_pe_record> all((size_t)n * per);
  std::vector<int> cnt(n, 0);
  const u32 max_tasks = n / 5000 + 2;
  std::vector<u32> st(max_tasks), en(max_tasks);
  const int nt = orc_ref_task_chunks(n, st.data(), en.data(), max_tasks);
#pragma omp parallel for schedule(dynamic, 1) num_threads(n_threads > 0 ? n_threads : 1)
  for (int t = 0; t < nt; ++t) {
    std::mt19937 gen(11);  // firstprivate copy per task
    for (u32 i = st[t]; i < en[t]; ++i)
      cnt[i] = map_one_pair(m->P, *m->ix, *m->ref, gen, seq1 + off1[i], off1[i + 1] - off1[i], seq2 + off2[i],
                            off2[i + 1] - off2[i], first_read_id + i, i, &all[(size_t)i * per], per, trace ? trace + i : nullptr);
  }
  int64_t n_out = 0;
  for (u32 i = 0; i < n; ++i) for (int j = 0; j < cnt[i] && n_out < cap_out; ++j) out[n_out++] = all[(size_t)i * per + j];
  return n_out;
}

static inline void tn5(orc_pe_record &r);
static inline void tn5_se(orc_pe_record &r);
void orc_mapper_set_barcodes(orc_mapper *m, const orc_whitelist *wl, int err_threshold, double prob_threshold, int output_not_in_whitelist) {
  m->wl = wl; m->bc_err_threshold = err_threshold; m->bc_prob_threshold = prob_threshold; m->output_not_in_whitelist = output_not_in_whitelist;
}

orc_whitelist *orc_whitelist_load(const char *path, uint32_t bc_len) {  // chromap.cc:388-431
  gzFile f = gzopen(path, "r");
  if (!f) return nullptr;
  orc_whitelist *wl = new orc_whitelist;
  wl->bc_len = bc_len;
  char buf[256];
  while (gzgets(f, buf, sizeof(buf)) != NULL) {
    size_t l = strlen(buf);
    if (l && buf[l - 1] == '\n') buf[--l] = 0;
    if (l != bc_len) { gzclose(f); delete wl; return nullptr; }
    wl->keys.push_back(barcode_seed(buf, l));
  }
  gzclose(f);
  std::sort(wl->keys.begin(), wl->keys.end());
  wl->keys.erase(std::unique(wl->keys.begin(), wl->keys.end()), wl->keys.end());
  wl->counts.assign(wl->keys.size(), 0);
  return wl;
}
void orc_whitelist_free(orc_whitelist *wl) { delete wl; }
// ComputeBarcodeAbundance (chromap.cc:492-548) over barcodes given in memory: n barcodes of bc_len bytes, in file
// order; `batch` = reference batch size (500000); sampling stops after the batch in which num_sample reaches `max_sample`.
void orc_whitelist_sample(orc_whitelist *wl, const char *bcs, uint64_t n, uint32_t bc_len, uint64_t max_sample, uint32_t batch) {
  for (uint64_t b0 = 0; b0 < n; b0 += batch) {
    const uint64_t b1 = std::min<uint64_t>(n, b0 + batch);
    for (uint64_t i = b0; i < b1; ++i) {
      const char *s = bcs + i * bc_len;
      bool has_n = false;
      for (u32 j = 0; j < bc_len; ++j) if (s[j] == 'N') has_n = true;
      if (has_n) continue;
      const int f = wl->find(barcode_seed(s, bc_len));
      if (f >= 0) { wl->counts[f] += 1; ++wl->num_sample; }
    }
    if (wl->num_sample >= max_sample) break;
  }
}
uint64_t orc_whitelist_arrays(const orc_whitelist *wl, const uint64_t **keys, const uint32_t **counts, uint64_t *num_sample) {
  *keys = wl->keys.data(); *counts = wl->counts.data(); *num_sample = wl->num_sample;
  return wl->keys.size();
}

// scATAC variant of the taskloop body: CorrectBarcodeAt first (chromap.h:897-909), the (corrected) barcode key
// travels with every record (mapping_generator.h:566-573).  bcs / quals: n * bc_len bytes each; out_bc[i] = barcode key
// of record i; bc_stats[0] += #barcodes in whitelist, bc_stats[1] += #corrected.
int64_t orc_map_pairs_bc(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2, const uint32_t *off2,
                         const char *bcs, const char *quals, uint32_t bc_len, uint32_t first_read_id, orc_pe_record *out, uint64_t *out_bc,
                         int64_t cap_out, int n_threads, uint64_t *bc_stats) {
  const int per = m->P.max_num_best_mappings;
  std::vector<orc_pe_record> all((size_t)n * per);
  std::vector<u64> keys(n, 0);
  std::vector<int> cnt(n, 0);
  const u32 max_tasks = n / 5000 + 2;
  std::vector<u32> st(max_tasks), en(max_tasks);
  const int nt = orc_ref_task_chunks(n, st.data(), en.data(), max_tasks);
  u64 n_in = 0, n_cor = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads(n_threads > 0 ? n_threads : 1) reduction(+ : n_in, n_cor)
  for (int t = 0; t < nt; ++t) {
    std::mt19937 gen(11);
    for (u32 i = st[t]; i < en[t]; ++i) {
      std::string bc(bcs + (size_t)i * bc_len, bc_len);
      bool ok = true;
      if (m->wl) ok = correct_barcode(*m->wl, m->bc_err_threshold, m->bc_prob_threshold, &bc[0], quals + (size_t)i * bc_len, bc_len, &n_in, &n_cor);
      keys[i] = barcode_seed(bc.data(), bc_len);
      if (!(ok || m->output_not_in_whitelist)) continue;
      cnt[i] = map_one_pair(m->P, *m->ix, *m->ref, gen, seq1 + off1[i], off1[i + 1] - off1[i], seq2 + off2[i], off2[i + 1] - off2[i],
                            first_read_id + i, i, &all[(size_t)i * per], per, nullptr);
    }
  }
  if (bc_stats) { bc_stats[0] += n_in; bc_stats[1] += n_cor; }
  int64_t n_out = 0;
  for (u32 i = 0; i < n; ++i)
    for (int j = 0; j < cnt[i] && n_out < cap_out; ++j) { out[n_out] = all[(size_t)i * per + j]; out_bc[n_out] = keys[i]; ++n_out; }
  return n_out;
}

// Post-processing with cell barcodes (PairedEndMappingWithBarcode, bed_mapping.h:116-167: order (start, len, barcode,
// mapq, ...), duplicates = same (barcode, start, len) — the atac preset dedups at cell level,
// remove_pcr_duplicates_at_bulk_level = false, chromap_driver.cc:256).
int64_t orc_postprocess_bc(const orc_params *p, orc_pe_record *recs, uint64_t *bcs, int64_t n) {
  if (n == 0) return 0;
  std::vector<int64_t> ord(n);
  std::iota(ord.begin(), ord.end(), 0);
  auto key = [&](int64_t i) {
    const orc_pe_record &r = recs[i];
    return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, bcs[i], r.mapq, r.direction, r.is_unique, r.read_id);
  };
  std::vector<orc_pe_record> rr(recs, recs + n);
  std::vector<u64> bb(bcs, bcs + n);
  if (!p->low_memory_mode && p->tn5_shift) for (auto &r : rr) { if (p->single_end) tn5_se(r); else tn5(r); }
  auto key2 = [&](int64_t i) {
    const orc_pe_record &r = rr[i];
    return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, bb[i], r.mapq, r.direction, r.is_unique, r.read_id);
  };
  (void)key;
  std::sort(ord.begin(), ord.end(), [&](int64_t a, int64_t b) { return key2(a) < key2(b); });
  const bool se = p->single_end != 0;  // MappingWithBarcode::operator== is (barcode, start) (bed_mapping.h:36-39)
  auto same = [&](int64_t a, int64_t b) {
    return rr[a].rid == rr[b].rid && rr[a].fragment_start == rr[b].fragment_start && (se || rr[a].fragment_length == rr[b].fragment_length) && bb[a] == bb[b];
  };
  int64_t o = 0, i = 0;
  while (i < n) {
    int64_t j = i + 1;
    int64_t keep = ord[i];
    u32 dups = 1;
    if (p->remove_pcr_duplicates)
      for (; j < n && same(ord[j], ord[j - 1]); ++j) {  // consecutive equality, as the merge / the in-memory pass compare
        ++dups;
        if (p->low_memory_mode) { if (rr[ord[j]].mapq > rr[keep].mapq) keep = ord[j]; }
        else keep = ord[j];  // in-memory dedup keeps the last of the run (mapping_processor.h:181-197)
      }
    orc_pe_record k = rr[keep];
    if (k.mapq >= p->mapq_threshold) {
      if (p->remove_pcr_duplicates) k.num_dups = std::min<u32>(255, dups);
      if (p->low_memory_mode && p->tn5_shift) { if (se) tn5_se(k); else tn5(k); }
      recs[o] = k; bcs[o] = bb[keep]; ++o;
    }
    i = j;
  }
  return o;
}

int64_t orc_format_bed_bc(const orc_reference *ref, const orc_pe_record *recs, const uint64_t *bcs, int64_t n, uint32_t bc_len, char *buf, int64_t cap) {
  int64_t len = 0;
  static const char tab[4] = {'A', 'C', 'G', 'T'};
  for (int64_t i = 0; i < n; ++i) {  // mapping_writer.cc:127-137, barcode_translator.h:114-123
    const orc_pe_record &r = recs[i];
    std::string line = ref->names[r.rid] + "\t" + std::to_string(r.fragment_start) + "\t" + std::to_string((u32)(r.fragment_start + r.fragment_length)) + "\t";
    for (u32 j = 0; j < bc_len; ++j) line.push_back(tab[(bcs[i] >> ((bc_len - 1 - j) * 2)) & 3]);
    line += "\t" + std::to_string((u32)r.num_dups) + "\n";
    if (buf && len + (int64_t)line.size() <= cap) memcpy(buf + len, line.data(), line.size());
    len += line.size();
  }
  return len;
}

// Whole-file scATAC driver: `chromap --preset atac -x idx -r ref -1 r1 -2 r2 -b bc [--barcode-whitelist wl] -o out`.
int orc_run_files_bc(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                     const char *barcode_path, const char *whitelist_path, const char *out_path, int n_threads, uint64_t *bc_stats) {
  orc_reference *ref = orc_reference_load(ref_path);
  orc_index *ix = orc_index_load(index_path);
  if (!ref || !ix) return -1;
  orc_mapper *m = orc_mapper_create(p, ix, ref);
  if (!m) return -2;
  // barcode length from the first records (chromap.cc:364-386), whitelist + abundance pre-pass (chromap.h:755-761)
  std::string allbc, allq;
  u32 bc_len = 0;
  {
    SeqReader rb;
    if (!rb.open(barcode_path)) return -3;
    std::string n, s, q;
    while (rb.next(n, s, q)) { if (s.empty()) continue; if (!bc_len) bc_len = s.size(); if (s.size() != bc_len) return -6; allbc += s; q.resize(bc_len, 'I'); allq += q; }
    rb.close();
  }
  orc_whitelist *wl = nullptr;
  if (whitelist_path && whitelist_path[0]) {
    wl = orc_whitelist_load(whitelist_path, bc_len);
    if (!wl) return -7;
    orc_whitelist_sample(wl, allbc.data(), allbc.size() / bc_len, bc_len, 20000000, 500000);
    orc_mapper_set_barcodes(m, wl, 1, 0.9, 0);
  }
  SeqReader r1, r2;
  if (!r1.open(read1_path) || !r2.open(read2_path)) return -3;
  std::vector<orc_pe_record> recs;
  std::vector<u64> rbc;
  const u32 batch = 500000;
  u32 read_id = 0;
  for (;;) {
    std::string s1, s2;
    std::vector<u32> o1{0}, o2{0};
    std::string n, s, q;
    u32 cnt = 0;
    while (cnt < batch) {
      bool a = r1.next(n, s, q);
      while (a && s.empty()) a = r1.next(n, s, q);
      if (!a) break;
      s1 += s; o1.push_back(s1.size());
      bool b = r2.next(n, s, q);
      while (b && s.empty()) b = r2.next(n, s, q);
      if (!b) return -4;
      s2 += s; o2.push_back(s2.size());
      ++cnt;
    }
    if (cnt == 0) break;
    if ((size_t)(read_id + cnt) * bc_len > allbc.size()) return -4;
    const size_t base = recs.size();
    recs.resize(base + (size_t)cnt * p->max_num_best_mappings);
    rbc.resize(recs.size());
    const int64_t got = orc_map_pairs_bc(m, cnt, s1.data(), o1.data(), s2.data(), o2.data(), allbc.data() + (size_t)read_id * bc_len,
                                         allq.data() + (size_t)read_id * bc_len, bc_len, read_id, recs.data() + base, rbc.data() + base,
                                         recs.size() - base, n_threads, bc_stats);
    recs.resize(base + got); rbc.resize(base + got);
    read_id += cnt;
  }
  r1.close(); r2.close();
  const int64_t keep = orc_postprocess_bc(p, recs.data(), rbc.data(), recs.size());
  const int64_t bytes = orc_format_bed_bc(ref, recs.data(), rbc.data(), keep, bc_len, nullptr, 0);
  std::vector<char> text(bytes + 1);
  orc_format_bed_bc(ref, recs.data(), rbc.data(), keep, bc_len, text.data(), bytes);
  FILE *f = fopen(out_path, "wb");
  if (!f) return -5;
  fwrite(text.data(), 1, bytes, f);
  fclose(f);
  orc_mapper_free(m); orc_index_free(ix); orc_reference_free(ref);
  if (wl) orc_whitelist_free(wl);
  return 0;
}

static inline auto rec_key(const orc_pe_record &r) {  // bed_mapping.h:208-215, prefixed by rid
  return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, r.mapq, r.direction, r.is_unique, r.read_id,
                         r.positive_alignment_length, r.negative_alignment_length);
}
static inline void tn5(orc_pe_record &r) {  // bed_mapping.h:225-230
  r.fragment_start += 4; r.positive_alignment_length -= 4; r.fragment_length -= 9; r.negative_alignment_length -= 5;
}

int64_t orc_postprocess(const orc_params *p, orc_pe_record *recs, int64_t n) {
  if (n == 0) return 0;
  auto less = [](const orc_pe_record &a, const orc_pe_record &b) { return rec_key(a) < rec_key(b); };
  auto same = [](const orc_pe_record &a, const orc_pe_record &b) {
    return a.rid == b.rid && a.fragment_start == b.fragment_start && a.fragment_length == b.fragment_length;
  };
  int64_t o = 0;
  if (p->low_memory_mode) {  // mapping_writer.h:166-376: merge == global sort; dedup; MAPQ filter; Tn5 last
    std::sort(recs, recs + n, less);
    int64_t i = 0;
    while (i < n) {
      orc_pe_record keep = recs[i];
      u32 dups = 1;
      int64_t j = i + 1;
      if (p->remove_pcr_duplicates)
        for (; j < n && same(recs[j], recs[i]); ++j) { ++dups; if (recs[j].mapq > keep.mapq) keep = recs[j]; }
      if (keep.mapq >= p->mapq_threshold) {
        keep.num_dups = std::min<u32>(255, dups);
        if (p->tn5_shift) tn5(keep);
        recs[o++] = keep;
      }
      i = j;
    }
    return o;
  }
  // chromap.h:1322-1355: Tn5 first, then sort (+ dedup keeping the last of each run), MAPQ filter at output
  if (p->tn5_shift) for (int64_t i = 0; i < n; ++i) tn5(recs[i]);
  std::sort(recs, recs + n, less);
  if (p->remove_pcr_duplicates) {
    int64_t i = 0, w = 0;
    while (i < n) {
      int64_t j = i + 1;
      while (j < n && same(recs[j], recs[i])) ++j;
      orc_pe_record keep = recs[j - 1];
      keep.num_dups = std::min<u32>(255, (u32)(j - i));
      recs[w++] = keep;
      i = j;
    }
    n = w;
  }
  for (int64_t i = 0; i < n; ++i) if (recs[i].mapq >= p->mapq_threshold) recs[o++] = recs[i];
  return o;
}

int64_t orc_format_bed(const orc_reference *ref, const orc_pe_record *recs, int64_t n, char *buf, int64_t cap) {
  int64_t len = 0;
  char line[512];
  for (int64_t i = 0; i < n; ++i) {  // mapping_writer.cc:75-83
    const orc_pe_record &r = recs[i];
    const int l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t%c\t%u\n", ref->names[r.rid].c_str(), r.fragment_start,
                           (u32)(r.fragment_start + r.fragment_length), (u32)r.mapq, r.direction ? '+' : '-', (u32)r.num_dups);
    if (buf && len + l <= cap) memcpy(buf + len, line, l);
    len += l;
  }
  return len;
}

int64_t orc_postprocess_pairs(const orc_params *p, orc_pairs_record *recs, int64_t n) {
  // records sit in the bucket of rid1; merge order = (bucket rid, PairsMapping::operator<) (pairs_mapping.h:40-43)
  std::sort(recs, recs + n, [](const orc_pairs_record &a, const orc_pairs_record &b) {
    return std::make_tuple(a.rid1, a.rid2, a.pos1, a.pos2, a.mapq, a.read_id) < std::make_tuple(b.rid1, b.rid2, b.pos1, b.pos2, b.mapq, b.read_id);
  });
  int64_t o = 0;
  if (p->remove_pcr_duplicates) {  // mapping_writer.h:234-300 with PairsMapping::operator==
    int64_t i = 0;
    while (i < n) {
      orc_pairs_record keep = recs[i];
      int64_t j = i + 1;
      for (; j < n && recs[j].rid1 == recs[i].rid1 && recs[j].pos1 == recs[i].pos1 && recs[j].rid2 == recs[i].rid2 && recs[j].pos2 == recs[i].pos2; ++j)
        if (recs[j].mapq > keep.mapq) keep = recs[j];
      if (keep.mapq >= p->mapq_threshold) recs[o++] = keep;
      i = j;
    }
    return o;
  }
  for (int64_t i = 0; i < n; ++i) if (recs[i].mapq >= p->mapq_threshold) recs[o++] = recs[i];
  return o;
}

int64_t orc_format_pairs(const orc_reference *ref, const orc_pairs_record *recs, int64_t n, const char *const *read_names,
                         uint32_t first_read_id, char *buf, int64_t cap) {
  int64_t len = 0;
  std::string hdr = "## pairs format v1.0.0\n#shape: upper triangle\n";
  for (size_t i = 0; i < ref->names.size(); ++i) hdr += "#chromsize: " + ref->names[i] + " " + std::to_string(ref->lens[i]) + "\n";
  hdr += "#columns: readID chrom1 pos1 chrom2 pos2 strand1 strand2 pair_type mapq1 mapq2\n";
  if (buf && (int64_t)hdr.size() <= cap) memcpy(buf, hdr.data(), hdr.size());
  len += hdr.size();
  for (int64_t i = 0; i < n; ++i) {
    const orc_pairs_record &r = recs[i];
    const std::string line = std::string(read_names[r.read_id - first_read_id]) + "\t" + ref->names[r.rid1] + "\t" + std::to_string(r.pos1 + 1) + "\t" +
                             ref->names[r.rid2] + "\t" + std::to_string(r.pos2 + 1) + "\t" + (r.strand1 ? "+" : "-") + "\t" + (r.strand2 ? "+" : "-") +
                             "\tUU\t" + std::to_string(r.mapq) + "\t" + std::to_string(r.mapq) + "\n";
    if (buf && len + (int64_t)line.size() <= cap) memcpy(buf + len, line.data(), line.size());
    len += line.size();
  }
  return len;
}

// --TagAlign for paired-end records (mapping_writer.cc:84-110): one line per mate, the duplicate count on the second
int64_t orc_format_tagalign(const orc_reference *ref, const orc_pe_record *recs, int64_t n, char *buf, int64_t cap) {
  int64_t len = 0;
  char line[1100];
  for (int64_t i = 0; i < n; ++i) {
    const orc_pe_record &r = recs[i];
    const u32 pos_end = r.fragment_start + r.positive_alignment_length, neg_end = r.fragment_start + r.fragment_length;
    const u32 neg_start = neg_end - r.negative_alignment_length;
    const char *nm = ref->names[r.rid].c_str();
    int l;
    if (r.direction)
      l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t+\n%s\t%u\t%u\tN\t%u\t-\t%u\n", nm, r.fragment_start, pos_end, (u32)r.mapq, nm, neg_start, neg_end,
                   (u32)r.mapq, (u32)r.num_dups);
    else
      l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t-\n%s\t%u\t%u\tN\t%u\t+\t%u\n", nm, neg_start, neg_end, (u32)r.mapq, nm, r.fragment_start, pos_end,
                   (u32)r.mapq, (u32)r.num_dups);
    if (buf && len + l <= cap) memcpy(buf + len, line, l);
    len += l;
  }
  return len;
}

int orc_run_files(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path,
                  const char *read2_path, const char *out_path, int n_threads, double *mapping_seconds, uint64_t *n_pairs_out) {
  orc_reference *ref = orc_reference_load(ref_path);
  orc_index *ix = orc_index_load(index_path);
  if (!ref || !ix) return -1;
  orc_mapper *m = orc_mapper_create(p, ix, ref);
  if (!m) return -2;
  SeqReader r1, r2;
  if (!r1.open(read1_path) || !r2.open(read2_path)) return -3;
  std::vector<orc_pe_record> recs;
  std::vector<std::string> names1;  // read-1 names, only kept for pairs output
  const bool pairs = p->output_format == 5;
  const u32 batch = 500000;  // chromap.h:182
  u32 read_id = 0;
  double secs = 0;
  uint64_t total = 0;
  for (;;) {
    std::string s1, s2;
    std::vector<u32> o1{0}, o2{0};
    std::string n, s, q;
    u32 cnt = 0;
    while (cnt < batch) {
      bool a = r1.next(n, s, q);
      while (a && s.empty()) a = r1.next(n, s, q);  // sequence_batch.cc:28-31 skips empty reads
      if (!a) break;
      s1 += s; o1.push_back(s1.size());
      if (pairs) names1.push_back(n);
      bool b = r2.next(n, s, q);
      while (b && s.empty()) b = r2.next(n, s, q);
      if (!b) { fprintf(stderr, "Numbers of reads don't match!\n"); return -4; }
      s2 += s; o2.push_back(s2.size());
      ++cnt;
    }
    if (cnt == 0) break;
    const size_t base = recs.size();
    recs.resize(base + (size_t)cnt * p->max_num_best_mappings);
    auto t0 = std::chrono::steady_clock::now();
    int64_t got = orc_map_pairs_mt(m, cnt, s1.data(), o1.data(), s2.data(), o2.data(), read_id, recs.data() + base, recs.size() - base, n_threads, nullptr);
    secs += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    recs.resize(base + got);
    read_id += cnt;
    total += cnt;
  }
  r1.close(); r2.close();
  int64_t bytes;
  std::vector<char> text;
  if (pairs) {
    static_assert(sizeof(orc_pairs_record) == sizeof(orc_pe_record), "record sizes");
    orc_pairs_record *pr = reinterpret_cast<orc_pairs_record *>(recs.data());
    const int64_t keep = orc_postprocess_pairs(p, pr, recs.size());
    std::vector<const char *> nm;
    for (const auto &x : names1) nm.push_back(x.c_str());
    bytes = orc_format_pairs(ref, pr, keep, nm.data(), 0, nullptr, 0);
    text.resize(bytes + 1);
    orc_format_pairs(ref, pr, keep, nm.data(), 0, text.data(), bytes);
  } else {
    const int64_t keep = orc_postprocess(p, recs.data(), recs.size());
    bytes = orc_format_bed(ref, recs.data(), keep, nullptr, 0);
    text.resize(bytes + 1);
    orc_format_bed(ref, recs.data(), keep, text.data(), bytes);
  }
  FILE *f = fopen(out_path, "wb");
  if (!f) return -5;
  fwrite(text.data(), 1, bytes, f);
  fclose(f);
  if (mapping_seconds) *mapping_seconds = secs;
  if (n_pairs_out) *n_pairs_out = total;
  orc_mapper_free(m); orc_index_free(ix); orc_reference_free(ref);
  return 0;
}


// ---- single-end (MappingWithoutBarcode, bed_mapping.h:61-113) -----------------------------------------------
int64_t orc_map_reads_se(orc_mapper *m, uint32_t n, const char *seq, const uint32_t *off, uint32_t first_read_id, orc_pe_record *out,
                         int64_t cap_out, int n_threads) {
  const int per = m->P.max_num_best_mappings;
  std::vector<orc_pe_record> all((size_t)n * per);
  std::vector<int> cnt(n, 0);
#pragma omp parallel for schedule(dynamic, 1024) num_threads(n_threads > 0 ? n_threads : 1)
  for (int64_t i = 0; i < (int64_t)n; ++i)
    cnt[i] = map_one_read_se(m->P, *m->ix, *m->ref, seq + off[i], off[i + 1] - off[i], first_read_id + (u32)i, (u32)i, &all[(size_t)i * per], per);
  int64_t n_out = 0;
  for (u32 i = 0; i < n; ++i) for (int j = 0; j < cnt[i] && n_out < cap_out; ++j) out[n_out++] = all[(size_t)i * per + j];
  return n_out;
}

int64_t orc_map_reads_se_bc(orc_mapper *m, uint32_t n, const char *seq, const uint32_t *off, const char *bcs, const char *quals, uint32_t bc_len,
                            uint32_t first_read_id, orc_pe_record *out, uint64_t *out_bc, int64_t cap_out, int n_threads, uint64_t *bc_stats) {
  const int per = m->P.max_num_best_mappings;
  std::vector<orc_pe_record> all((size_t)n * per);
  std::vector<u64> keys(n, 0);
  std::vector<int> cnt(n, 0);
  u64 n_in = 0, n_cor = 0;
#pragma omp parallel for schedule(dynamic, 1024) num_threads(n_threads > 0 ? n_threads : 1) reduction(+ : n_in, n_cor)
  for (int64_t i = 0; i < (int64_t)n; ++i) {  // chromap.h:392-409: barcode gate first
    std::string bc(bcs + (size_t)i * bc_len, bc_len);
    bool ok = true;
    if (m->wl) ok = correct_barcode(*m->wl, m->bc_err_threshold, m->bc_prob_threshold, &bc[0], quals + (size_t)i * bc_len, bc_len, &n_in, &n_cor);
    keys[i] = barcode_seed(bc.data(), bc_len);
    if (!(ok || m->output_not_in_whitelist)) continue;
    cnt[i] = map_one_read_se(m->P, *m->ix, *m->ref, seq + off[i], off[i + 1] - off[i], first_read_id + (u32)i, (u32)i, &all[(size_t)i * per], per);
  }
  if (bc_stats) { bc_stats[0] += n_in; bc_stats[1] += n_cor; }
  int64_t n_out = 0;
  for (u32 i = 0; i < n; ++i)
    for (int j = 0; j < cnt[i] && n_out < cap_out; ++j) { out[n_out] = all[(size_t)i * per + j]; out_bc[n_out] = keys[i]; ++n_out; }
  return n_out;
}

static inline void tn5_se(orc_pe_record &r) {  // bed_mapping.h:97-103
  if (r.direction == 1) r.fragment_start += 4; else r.fragment_length -= 5;
}

// Order bed_mapping.h:83-88 (prefixed by rid), duplicates = same start on the same sequence (:89-92).
int64_t orc_postprocess_se(const orc_params *p, orc_pe_record *recs, int64_t n) {
  if (n == 0) return 0;
  auto key = [](const orc_pe_record &r) { return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, r.mapq, r.direction, r.is_unique, r.read_id); };
  auto less = [&](const orc_pe_record &a, const orc_pe_record &b) { return key(a) < key(b); };
  auto same = [](const orc_pe_record &a, const orc_pe_record &b) { return a.rid == b.rid && a.fragment_start == b.fragment_start; };
  int64_t o = 0;
  if (p->low_memory_mode) {  // mapping_writer.h:166-376
    std::sort(recs, recs + n, less);
    int64_t i = 0;
    while (i < n) {
      orc_pe_record keep = recs[i];
      u32 dups = 1;
      int64_t j = i + 1;
      if (p->remove_pcr_duplicates)
        for (; j < n && same(recs[j], recs[i]); ++j) { ++dups; if (recs[j].mapq > keep.mapq) keep = recs[j]; }
      if (keep.mapq >= p->mapq_threshold) {
        keep.num_dups = std::min<u32>(255, dups);
        if (p->tn5_shift) tn5_se(keep);
        recs[o++] = keep;
      }
      i = j;
    }
    return o;
  }
  if (p->tn5_shift) for (int64_t i = 0; i < n; ++i) tn5_se(recs[i]);  // chromap.h:594-597
  std::sort(recs, recs + n, less);
  if (p->remove_pcr_duplicates) {  // mapping_processor.h:161-202
    int64_t i = 0, w = 0;
    while (i < n) {
      int64_t j = i + 1;
      while (j < n && same(recs[j], recs[j - 1])) ++j;
      orc_pe_record keep = recs[j - 1];
      keep.num_dups = std::min<u32>(255, (u32)(j - i));
      recs[w++] = keep;
      i = j;
    }
    n = w;
  }
  for (int64_t i = 0; i < n; ++i) if (recs[i].mapq >= p->mapq_threshold) recs[o++] = recs[i];
  return o;
}

int orc_run_files_se(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *out_path,
                     int n_threads) {
  orc_reference *ref = orc_reference_load(ref_path);
  orc_index *ix = orc_index_load(index_path);
  if (!ref || !ix) return -1;
  orc_mapper *m = orc_mapper_create(p, ix, ref);
  if (!m) return -2;
  SeqReader r1;
  if (!r1.open(read1_path)) return -3;
  std::vector<orc_pe_record> recs;
  const u32 batch = 500000;
  u32 read_id = 0;
  for (;;) {
    std::string s1, n, s, q;
    std::vector<u32> o1{0};
    u32 cnt = 0;
    while (cnt < batch) {
      bool a = r1.next(n, s, q);
      while (a && s.empty()) a = r1.next(n, s, q);
      if (!a) break;
      s1 += s; o1.push_back(s1.size());
      ++cnt;
    }
    if (cnt == 0) break;
    const size_t base = recs.size();
    recs.resize(base + (size_t)cnt * p->max_num_best_mappings);
    const int64_t got = orc_map_reads_se(m, cnt, s1.data(), o1.data(), read_id, recs.data() + base, recs.size() - base, n_threads);
    recs.resize(base + got);
    read_id += cnt;
  }
  r1.close();
  const int64_t keep = orc_postprocess_se(p, recs.data(), recs.size());
  const int64_t bytes = orc_format_bed(ref, recs.data(), keep, nullptr, 0);
  std::vector<char> text(bytes + 1);
  orc_format_bed(ref, recs.data(), keep, text.data(), bytes);
  FILE *f = fopen(out_path, "wb");
  if (!f) return -5;
  fwrite(text.data(), 1, bytes, f);
  fclose(f);
  orc_mapper_free(m); orc_index_free(ix); orc_reference_free(ref);
  return 0;
}


// ---- SAM (oracle only, groundwork): chromap --SAM for bulk single-end / paired-end reads, non-split --------------------
int orc_run_files_sam(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                      const char *out_path) {
  orc_reference *ref = orc_reference_load(ref_path);
  orc_index *ix = orc_index_load(index_path);
  if (!ref || !ix || p->split_alignment) return -1;
  const bool se = !read2_path || !*read2_path;
  SeqReader r1, r2;
  if (!r1.open(read1_path) || (!se && !r2.open(read2_path))) return -3;
  std::vector<SamRec> recs;
  const u32 batch = 500000;
  u32 read_id = 0;
  for (;;) {
    std::vector<std::string> n1, s1, q1, n2, s2, q2;
    std::string n, s, q;
    while (n1.size() < batch) {
      bool a = r1.next(n, s, q);
      while (a && s.empty()) a = r1.next(n, s, q);
      if (!a) break;
      n1.push_back(n); s1.push_back(s); q1.push_back(q);
      if (!se) {
        bool b = r2.next(n, s, q);
        while (b && s.empty()) b = r2.next(n, s, q);
        if (!b) return -4;
        n2.push_back(n); s2.push_back(s); q2.push_back(q);
      }
    }
    const u32 cnt = (u32)n1.size();
    if (cnt == 0) break;
    std::vector<u32> st(cnt / 5000 + 2), en(cnt / 5000 + 2);
    const int nt = orc_ref_task_chunks(cnt, st.data(), en.data(), (int)st.size());
    orc_pe_record dummy[8];
    for (int t = 0; t < nt; ++t) {
      std::mt19937 gen(11);
      for (u32 i = st[t]; i < en[t]; ++i) {
        SamSink sink{&recs, n1[i].c_str(), q1[i].c_str(), se ? nullptr : n2[i].c_str(), se ? nullptr : q2[i].c_str()};
        if (se) map_one_read_se(*p, *ix, *ref, s1[i].data(), (u32)s1[i].size(), read_id + i, i, dummy, 8, &sink);
        else map_one_pair(*p, *ix, *ref, gen, s1[i].data(), (u32)s1[i].size(), s2[i].data(), (u32)s2[i].size(), read_id + i, i, dummy, 8, nullptr, &sink);
      }
    }
    read_id += cnt;
  }
  r1.close(); if (!se) r2.close();
  // SAMMapping::operator< (sam_mapping.h:188-193) prefixed by the bucket (= rid); operator== (:194-199)
  auto key = [](const SamRec &r) { return std::make_tuple(r.rid, r.pos, (u64)0, r.mrid, r.mpos, r.flag & 64, r.mapq, r.read_id); };
  std::stable_sort(recs.begin(), recs.end(), [&](const SamRec &a, const SamRec &b) { return key(a) < key(b); });
  auto same = [](const SamRec &a, const SamRec &b) { return a.rid == b.rid && a.pos == b.pos && (a.flag & 64) == (b.flag & 64) && a.mrid == b.mrid && a.mpos == b.mpos; };
  std::vector<const SamRec *> keep;
  if (p->remove_pcr_duplicates) {
    size_t i = 0;
    while (i < recs.size()) {
      size_t j = i + 1, k = i;
      for (; j < recs.size() && same(recs[j], recs[j - 1]); ++j) {
        if (p->low_memory_mode) { if (recs[j].mapq > recs[k].mapq) k = j; } else k = j;
      }
      keep.push_back(&recs[k]);
      i = j;
    }
  } else for (const auto &r : recs) keep.push_back(&r);
  FILE *f = fopen(out_path, "wb");
  if (!f) return -5;
  for (size_t i = 0; i < ref->names.size(); ++i) fprintf(f, "@SQ\tSN:%s\tLN:%u\n", ref->names[i].c_str(), ref->lens[i]);  // mapping_writer.cc:312-321
  for (const SamRec *r : keep) {  // mapping_writer.cc:324-356
    if (r->mapq < p->mapq_threshold) continue;
    std::string cig;
    for (u32 c : r->cigar) { cig += std::to_string(c >> 4); cig.push_back("MIDNSHP=XB"[c & 0xf]); }
    if (cig.empty()) cig = "*";
    const std::string mate = r->mrid < 0 ? "*" : (r->mrid == r->rid ? "=" : ref->names[r->mrid]);
    fprintf(f, "%s\t%d\t%s\t%lld\t%d\t%s\t%s\t%lld\t%d\t%s\t%s\tNM:i:%d\tMD:Z:%s\n", r->name.c_str(), r->flag, ref->names[r->rid].c_str(), (long long)r->pos + 1,
            r->mapq, cig.c_str(), mate.c_str(), r->mrid < 0 ? 0LL : (long long)r->mpos + 1, r->tlen, r->seq.c_str(), r->qual.c_str(), r->nm, r->md.c_str());
  }
  fclose(f);
  orc_index_free(ix); orc_reference_free(ref);
  return 0;
}


// test hook: the oracle's sg_align on raw buffers (checks the device-side restatement compiled for the host)
int orc_sg_align_test(const char *win, int wlen, const char *read, int rlen, int w, unsigned *cigar, int cap, int *start, int *end) {
  SamAln a;
  sg_align(win, wlen, read, rlen, 1, 4, 6, 1, 6, 1, w, a);
  *start = a.start; *end = a.end;
  int n = 0;
  for (u32 c : a.cigar) if (n < cap) cigar[n++] = c;
  return (int)a.cigar.size();
}


// SAM cores in the layout of cmx_sam_record (include/chromap_b200.h) for the device parity tests: one per reported pair
// (paired-end: seq2 != NULL) or read.
int64_t orc_map_sam_cores(orc_mapper *m, uint32_t n, const char *seq1, const uint32_t *off1, const char *seq2, const uint32_t *off2, uint32_t first_read_id,
                          orc_sam_record *out, int64_t cap_out) {
  std::vector<u32> st(n / 5000 + 2), en(n / 5000 + 2);
  const int nt = orc_ref_task_chunks(n, st.data(), en.data(), (int)st.size());
  const bool se = seq2 == nullptr;
  int64_t n_out = 0;
  orc_pe_record dummy[8];
  for (int t = 0; t < nt; ++t) {
    std::mt19937 gen(11);
    for (u32 i = st[t]; i < en[t]; ++i) {
      std::vector<SamRec> recs;
      SamSink sink{&recs, "", "", "", ""};
      if (se) map_one_read_se(m->P, *m->ix, *m->ref, seq1 + off1[i], off1[i + 1] - off1[i], first_read_id + i, i, dummy, 8, &sink);
      else map_one_pair(m->P, *m->ix, *m->ref, gen, seq1 + off1[i], off1[i + 1] - off1[i], seq2 + off2[i], off2[i + 1] - off2[i], first_read_id + i, i, dummy, 8, nullptr, &sink);
      const size_t per = se ? 1 : 2;
      for (size_t k = 0; k + per <= recs.size() && n_out < cap_out; k += per) {
        orc_sam_record &o = out[n_out++];
        memset(&o, 0, sizeof(o));
        o.read_id = recs[k].read_id; o.rid = (u32)recs[k].rid; o.mapq = (uint8_t)recs[k].mapq; o.is_unique = (uint8_t)recs[k].is_unique;
        o.secondary = (recs[k].flag & 256) ? 1 : 0;
        for (size_t q = 0; q < per; ++q) {
          const SamRec &r = recs[k + q];
          int ref_len = 0;
          for (u32 c : r.cigar) if ((c & 0xf) != 1) ref_len += c >> 4;
          o.pos[q] = (u32)r.pos; o.end[q] = (u32)r.pos + ref_len - 1; o.strand[q] = (uint8_t)r.strand_pos;
          o.n_cigar[q] = (uint8_t)std::min<size_t>(r.cigar.size(), ORC_SAM_MAX_CIGAR);
          for (size_t c = 0; c < o.n_cigar[q]; ++c) o.cigar[q][c] = r.cigar[c];
        }
      }
    }
  }
  return n_out;
}


// ---- PAF (oracle only, groundwork): chromap --PAF for bulk single-end / paired-end reads, non-split ---------------------
int orc_run_files_paf(const orc_params *p, const char *index_path, const char *ref_path, const char *read1_path, const char *read2_path,
                      const char *out_path) {
  orc_reference *ref = orc_reference_load(ref_path);
  orc_index *ix = orc_index_load(index_path);
  if (!ref || !ix || p->split_alignment) return -1;
  const bool se = !read2_path || !*read2_path;
  SeqReader r1, r2;
  if (!r1.open(read1_path) || (!se && !r2.open(read2_path))) return -3;
  std::vector<PafRec> recs;
  std::vector<SamRec> unused;
  const u32 batch = 500000;
  u32 read_id = 0;
  for (;;) {
    std::vector<std::string> n1, s1, n2, s2;
    std::string n, s, q;
    while (n1.size() < batch) {
      bool a = r1.next(n, s, q);
      while (a && s.empty()) a = r1.next(n, s, q);
      if (!a) break;
      n1.push_back(n); s1.push_back(s);
      if (!se) {
        bool b = r2.next(n, s, q);
        while (b && s.empty()) b = r2.next(n, s, q);
        if (!b) return -4;
        n2.push_back(n); s2.push_back(s);
      }
    }
    const u32 cnt = (u32)n1.size();
    if (cnt == 0) break;
    std::vector<u32> st(cnt / 5000 + 2), en(cnt / 5000 + 2);
    const int nt = orc_ref_task_chunks(cnt, st.data(), en.data(), (int)st.size());
    orc_pe_record dummy[8];
    for (int t = 0; t < nt; ++t) {
      std::mt19937 gen(11);
      for (u32 i = st[t]; i < en[t]; ++i) {
        SamSink sink{&unused, n1[i].c_str(), "", se ? "" : n2[i].c_str(), "", &recs};
        if (se) map_one_read_se(*p, *ix, *ref, s1[i].data(), (u32)s1[i].size(), read_id + i, i, dummy, 8, &sink);
        else map_one_pair(*p, *ix, *ref, gen, s1[i].data(), (u32)s1[i].size(), s2[i].data(), (u32)s2[i].size(), read_id + i, i, dummy, 8, nullptr, &sink);
      }
    }
    read_id += cnt;
  }
  r1.close(); if (!se) r2.close();
  auto tn5 = [&](PafRec &r) {  // paf_mapping.h: PAFMapping::Tn5Shift / PairedPAFMapping::Tn5Shift
    if (se) { if (r.dir == 1) r.start += 4; else r.frag -= 5; }
    else { r.start += 4; r.pal -= 4; r.frag -= 9; r.nal -= 5; }
  };
  if (!p->low_memory_mode && p->tn5_shift) for (auto &r : recs) tn5(r);
  auto key = [&](const PafRec &r) {
    return se ? std::make_tuple(r.rid, r.start, r.frag, (uint8_t)r.mapq, (uint8_t)0, r.dir, r.uniq, r.read_id, r.len1, (uint16_t)0)
              : std::make_tuple(r.rid, r.start, r.frag, r.mapq1, r.mapq2, r.dir, r.uniq, r.read_id, r.pal, r.nal);
  };
  std::stable_sort(recs.begin(), recs.end(), [&](const PafRec &a, const PafRec &b) { return key(a) < key(b); });
  auto same = [&](const PafRec &a, const PafRec &b) { return a.rid == b.rid && a.start == b.start && (se || a.frag == b.frag); };
  std::vector<PafRec> keep;
  size_t i = 0;
  while (i < recs.size()) {
    size_t j = i + 1, k = i;
    u32 dups = 1;
    if (p->remove_pcr_duplicates)
      for (; j < recs.size() && same(recs[j], recs[j - 1]); ++j) {
        ++dups;
        if (p->low_memory_mode) { if (recs[j].mapq > recs[k].mapq) k = j; } else k = j;
      }
    PafRec r = recs[k];
    if (p->remove_pcr_duplicates || p->low_memory_mode) r.dups = (uint8_t)std::min<u32>(255, dups);
    if (r.mapq >= p->mapq_threshold) { if (p->low_memory_mode && p->tn5_shift) tn5(r); keep.push_back(r); }
    i = j;
  }
  FILE *f = fopen(out_path, "wb");
  if (!f) return -5;
  for (const PafRec &r : keep) {  // mapping_writer.cc:177-196 (single-end), :249-310 (paired-end)
    const char *rn = ref->names[r.rid].c_str();
    const u32 rl = ref->lens[r.rid];
    if (se) {
      fprintf(f, "%s\t%u\t0\t%u\t%c\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", r.name1.c_str(), (u32)r.len1, (u32)r.len1, r.dir ? '+' : '-', rn, rl, r.start,
              (u32)(r.start + r.frag), (u32)r.len1, (u32)r.frag, (u32)r.mapq);
      continue;
    }
    const u32 pos_end = r.start + r.pal, neg_end = r.start + r.frag, neg_start = neg_end - r.nal;
    if (r.dir) {
      fprintf(f, "%s\t%u\t0\t%u\t+\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", r.name1.c_str(), (u32)r.len1, (u32)r.len1, rn, rl, r.start, pos_end, (u32)r.len1, (u32)r.pal, (u32)r.mapq1);
      fprintf(f, "%s\t%u\t0\t%u\t-\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", r.name2.c_str(), (u32)r.len2, (u32)r.len2, rn, rl, neg_start, neg_end, (u32)r.len2, (u32)r.nal, (u32)r.mapq2);
    } else {
      fprintf(f, "%s\t%u\t0\t%u\t-\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", r.name1.c_str(), (u32)r.len1, (u32)r.len1, rn, rl, neg_start, neg_end, (u32)r.len1, (u32)r.nal, (u32)r.mapq1);
      fprintf(f, "%s\t%u\t0\t%u\t+\t%s\t%u\t%u\t%u\t%u\t%u\t%u\n", r.name2.c_str(), (u32)r.len2, (u32)r.len2, rn, rl, r.start, pos_end, (u32)r.len2, (u32)r.pal, (u32)r.mapq2);
    }
  }
  fclose(f);
  orc_index_free(ix); orc_reference_free(ref);
  return 0;
}

}  // extern "C"
