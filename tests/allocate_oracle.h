// Test infrastructure: a restatement of the reference's AllocateMultiMappings (mapping_processor.h:204-440) on records that are
// already sorted and deduplicated (the oracle's in-memory post-processing with the MAPQ filter at 0).  The overlap count walks
// an implicit augmented interval tree over each sequence's uni records, as the reference does, and not the binary-search
// formula of the library, so that the device count is checked against an independent form.  The draw is libstdc++'s own
// std::discrete_distribution on std::mt19937.  Header-only: included by the emulated test, built into a small shared object
// by the oracle test.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <random>
#include <vector>

struct orc_alloc_record {  // cmx_pe_record / orc_pe_record
  uint32_t read_id, rid, fragment_start;
  uint16_t fragment_length;
  uint8_t mapq, direction, is_unique, num_dups;
  uint16_t positive_alignment_length, negative_alignment_length;
};
struct orc_alloc_stats {
  uint64_t n_multi, n_allocated, n_without_overlap, n_draws, n_uni_after, n_multi_after;
};

// Implicit augmented interval tree: node i of a sorted array sits at level = number of trailing 1 bits of i; max_end[i] is
// the largest end in its subtree.  Nodes at or past n exist only as placeholders on the path to the root.
struct OrcIntervalTree {
  std::vector<uint32_t> start, end, max_end;
  int root_level = 0;
  void build() {
    const size_t n = start.size();
    max_end.assign(n, 0);
    for (size_t i = 0; i < n; i += 2) max_end[i] = end[i];
    if (n == 0) { root_level = 0; return; }
    size_t last_i = 0;
    uint32_t last = 0;
    for (size_t i = 0; i < n; i += 2) { last_i = i; last = end[i]; }
    int k = 1;
    for (; ((size_t)1 << k) <= n; ++k) {
      const size_t x = (size_t)1 << (k - 1), first = (x << 1) - 1, step = x << 2;
      for (size_t i = first; i < n; i += step) {
        const uint32_t left = max_end[i - x], right = i + x < n ? max_end[i + x] : last;
        max_end[i] = std::max(end[i], std::max(left, right));
      }
      last_i = (last_i >> k & 1) ? last_i - x : last_i + x;
      if (last_i < n && max_end[last_i] > last) last = max_end[last_i];
    }
    root_level = k - 1;
  }
  // number of intervals with start < qe && qs < end
  uint32_t count(uint32_t qs, uint32_t qe) const {
    const size_t n = start.size();
    struct Cell { int level; size_t node; bool left_done; };
    Cell stack[64];
    int top = 0;
    uint32_t c = 0;
    stack[top++] = {root_level, ((size_t)1 << root_level) - 1, false};
    while (top) {
      const Cell z = stack[--top];
      if (z.level <= 3) {  // a small subtree: scan it in order
        const size_t lo = z.node >> z.level << z.level;
        const size_t hi = std::min(n, lo + ((size_t)1 << (z.level + 1)) - 1);
        for (size_t i = lo; i < hi && start[i] < qe; ++i) c += qs < end[i];
      } else if (!z.left_done) {
        const size_t left = z.node - ((size_t)1 << (z.level - 1));
        stack[top++] = {z.level, z.node, true};
        if (left >= n || max_end[left] > qs) stack[top++] = {z.level - 1, left, false};
      } else if (z.node < n && start[z.node] < qe) {
        c += qs < end[z.node];
        stack[top++] = {z.level - 1, z.node + ((size_t)1 << (z.level - 1)), false};
      }
    }
    return c;
  }
};

// recs[0, n) sorted and deduplicated; keep[i] = 1 for the records that survive the allocation.  Returns -1 (the reference
// aborts) when there is no multi-mapping, else 0.
static inline int orc_allocate_flags(const orc_alloc_record *recs, uint64_t n, uint32_t n_seq, int32_t distance, int32_t seed, uint8_t *keep,
                                     orc_alloc_stats *st) {
  std::vector<OrcIntervalTree> trees(n_seq);
  std::vector<uint64_t> multi;  // record index, in (rid, record) order
  for (uint64_t i = 0; i < n; ++i) {
    keep[i] = 0;
    if (recs[i].mapq < 4) { multi.push_back(i); continue; }
    keep[i] = 1;
    trees[recs[i].rid].start.push_back(recs[i].fragment_start);
    trees[recs[i].rid].end.push_back(recs[i].fragment_start + recs[i].fragment_length);
  }
  for (auto &t : trees) t.build();
  *st = orc_alloc_stats{};
  st->n_multi = multi.size();
  if (multi.empty()) return -1;
  std::stable_sort(multi.begin(), multi.end(), [&](uint64_t a, uint64_t b) { return recs[a].read_id < recs[b].read_id; });
  std::mt19937 generator(seed);
  const uint32_t d = (uint32_t)distance;
  std::vector<uint32_t> w;
  for (size_t s = 0; s < multi.size();) {
    size_t e = s;
    uint32_t sum = 0;
    w.clear();
    for (; e < multi.size() && recs[multi[e]].read_id == recs[multi[s]].read_id; ++e) {
      const orc_alloc_record &r = recs[multi[e]];
      const uint32_t start = r.fragment_start, end = start + r.fragment_length;
      w.push_back(trees[r.rid].count(start > d ? start - d : 0u, end + d));
      sum += w.back();
    }
    if (sum == 0) ++st->n_without_overlap;
    else {
      std::discrete_distribution<uint32_t> dist(w.begin(), w.end());
      keep[multi[s + dist(generator)]] = 1;
      ++st->n_allocated;
      st->n_draws += w.size() >= 2;
    }
    s = e;
  }
  for (uint64_t i = 0; i < n; ++i)
    if (keep[i]) { if (recs[i].is_unique == 1) ++st->n_uni_after; else ++st->n_multi_after; }
  return 0;
}
