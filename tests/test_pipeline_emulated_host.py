"""The whole device pipeline — seed_front -> cluster -> pair_candidates -> verify -> pairing (tier 0, thread kernels), prep ->
seed_cta -> pair_candidates_cta -> verify_cta -> pairing_cta (overflow tiers, one CTA per read / pair), overflow collection
between the tiers, select, emit (+ deferred tracebacks) / emit_cta — compiled from the UNCHANGED kernel sources
(device_common.cuh, minimizers.cuh, pipeline_kernels.cuh, seed_front.cuh, cta_pair_candidates.cuh, cta_verify_pairing.cuh, sam_kernels.cuh) and run on the host
emulation of CTAs (tests/cta_emu.h) by the library's own launch sequence (lane_pipeline.cuh: kernel order, grid / block and
shared-memory sizes, the host decisions between the kernels) and scratch layout (`scratch_layout`), against the oracle's mapper
(`orc_map_pairs`, pinned to the reference binary by tests/test_oracle_golden.py): every pair's records, field by field.
The front end runs too (seed_front_kernel: persistent grid, double-buffered read tiles, packed-key minimizer scan, table probes,
lane-interleaved records): only its six PTX wrappers (mbarrier.* / cp.async.bulk) are replaced by cta_emu.h's host equivalents —
an mbarrier word with byte and arrival counts, a copy that signals its bytes — and its records are also compared one by one with
the oracle's minimizers and khash lookups.
Runs: `--preset chip` with the real tier capacities (64 / 32 / 32 ...) on a reference with repeat families, reads longer than the first tier
allows, N's and junk pairs; and tiny first- and second-tier capacities that push most ordinary pairs through the CTA kernels and
some of them up to the last tier (512-thread pair_candidates_cta, 256-thread verify_cta), with -n 3; `--preset atac` (adapter
trimming by prep_kernel on read-through pairs); `--preset hic` (split alignment: verify_split / pairing_split / emit_split and the
CTA form, chimeric reads, pairs records); single-end (emit_se_kernel, a fresh generator per read), each also through the CTA tiers; `--SAM` (emit_sam_kernel: spans and CIGARs by
the diagonal-band aligner, against the oracle's SAM cores); a 420-copy repeat family (thousands of hits and hundreds of candidates per
read, the real capacities up to the last tier).  The whole pipeline also runs at index shapes (19, 10), (23, 11) (k > 22: no
shared-memory key buffer in the front end; chip, CTA tiers, single-end, SAM, Hi-C), (28, 20) and (16, 5), and at mapping knobs
off their defaults: -e 1 / 7 / 15, -n 8 through the CTA tiers, -s 1, -f low enough for repetitive seeds and the second seeding
round, --drop-repetitive-reads and --min-read-length."""
import os
import re
import subprocess

from tests import emu

MAIN = r'''
extern "C" {
#include "%(orc_h)s"
}
struct HostTier {
  Caps caps;
  std::vector<char> mem;
  std::vector<std::vector<char>> parts;   // EMU_EXACT_SCRATCH: every scratch array its own exactly sized allocation (AddressSanitizer then sees overruns between them)
  Scratch view;
};
static void tier_prepare_host(HostTier &t, int n_slots, const int *pair_list, bool interleaved) {
  size_t o[SCRATCH_ARRAYS];
  const size_t bytes = scratch_layout(t.caps, (size_t)n_slots + 1, interleaved, o);
  t.mem.assign(bytes + 256, (char)0x5A);   // (scratch is not cleared on the device either)
  char *a[SCRATCH_ARRAYS];
  for (int i = 0; i < SCRATCH_ARRAYS; ++i) a[i] = t.mem.data() + o[i];
  if (getenv("EMU_EXACT_SCRATCH")) {
    size_t sz[SCRATCH_ARRAYS];
    scratch_layout(t.caps, (size_t)n_slots, interleaved, o, sz);
    t.parts.assign(SCRATCH_ARRAYS, std::vector<char>());
    for (int i = 0; i < SCRATCH_ARRAYS; ++i) { t.parts[(size_t)i].assign(sz[i] ? sz[i] : 8, (char)0x5A); a[i] = t.parts[(size_t)i].data(); }
  }
  Scratch &S = t.view;
  S.caps = t.caps; S.n_slots = n_slots; S.pair_list = pair_list; S.mm_il = interleaved ? 1 : 0;
  scratch_bind(S, a);
}
static std::vector<u64> g_smem;
// The emulation's side of the library's launch sequence (lane_pipeline.cuh): a launch runs the grid's CTAs one after the
// other.  Dynamic shared memory and the list buffers are fresh allocations of exactly the size asked for, so that
// AddressSanitizer sees any access past them.
struct EmuLane {
  HostTier tiers[N_TIERS];
  std::vector<char> lists[LIST_OVERFLOW + N_TIERS];
  int cnt[4] = {0, 0, 0, 0};
  std::vector<int> chunks;
  size_t max_smem = 0;   // the largest dynamic shared memory a launch asked for
  int cluster_launches = 0;
  template <typename... KA, typename... A>
  void operator()(void (*kernel)(KA...), int grid, int block, size_t smem, A... a) {
    max_smem = std::max(max_smem, smem);
    if ((void *)kernel == (void *)&cluster_kernel) ++cluster_launches;
    g_smem = std::vector<u64>((smem + 7) / 8, 0xA5A5A5A5A5A5A5A5ull);
    g_dyn_smem = g_smem.data();
    emu_grid(grid, block, [&]() { kernel(a...); });
  }
  void mark(int) {}
  void wait_piece(u32) {}
  Scratch tier(int t, int n, const int *pair_list) { tier_prepare_host(tiers[t], n, pair_list, t == 0); return tiers[t].view; }
  void *list(int l, size_t bytes) { lists[l] = std::vector<char>(bytes); return lists[l].data(); }
  void clear_counts(int i, int n) { std::fill(cnt + i, cnt + i + n, 0); }
  int overflow_count(int) { return cnt[0]; }
  const int *sort_list(int *list, int n) { std::sort(list, list + n); return list; }
  const int *chunk_starts(const std::vector<int> &c) { chunks = c; return chunks.data(); }
  void emit_on(int) {}
  void emit_join(int) {}
};
static char comp(char c) { switch (c) { case 'A': case 'a': return 'T'; case 'C': case 'c': return 'G'; case 'G': case 'g': return 'C'; case 'T': case 't': return 'A'; default: return 'N'; } }
static std::string revc(const std::string &s) { std::string r(s.rbegin(), s.rend()); for (auto &c : r) c = comp(c); return r; }

struct RunStats {
  long pairs = 0, records = 0, tier_pairs[3] = {0, 0, 0}, bad = 0;
  // oracle records at the ends of reference sequences (runs with `edges`): starting within L + e of the start of a rid > 0, ending
  // within e + 1 of a sequence's end, on a sequence shorter than 2L; and pairs whose mate-guided lookup ran with a window that begins
  // below the start of a rid > 0 (`lookup_at_start`: a mate without candidates of its own mapped by the lookup, the whole fragment
  // within 2 * max_insert of the rid's start, so the partner's candidate lies there too)
  long edge_start = 0, edge_end = 0, short_seq = 0, lookup_at_start = 0;
  // front-end tiles (per mate) too long to stage, read by each thread from global memory (seed_front_kernel's own test
  // g1 - base > tb); reads that cluster_kernel's first pass listed for the second; reads of mapped pairs with 256 or more
  // minimizers (the oracle's count: candidate counts are u8 and wrap there); the launches' largest dynamic shared memory
  long unstaged = 0, second_pass = 0, mm256 = 0, max_smem = 0, cluster_launches = 0;
  // runs with `bytes`: oracle records whose read 1 has a lower-case base, by that read's strand field (0 / 1)
  long lower_s0 = 0, lower_s1 = 0;
};

enum { MODE_CHIP = 0, MODE_ATAC = 1, MODE_HIC = 2, MODE_SE = 3, MODE_SAM = 4, MODE_SAM_SE = 5 };
// mapping knobs over the preset (-1: the preset's value): -e, -s, -f f0,f1, --drop-repetitive-reads, --min-read-length
struct Knobs { int e = -1, min_seeds = -1, f0 = -1, f1 = -1, drop_rep = -1, min_read_len = -1; };
static RunStats run_case(int mode, int seed, int n_pairs, int mrl, const Caps *caps3, int max_best, int read_len_base, bool front_only = false, int K = 17, int W = 7, int fam_copies = 90,
                         const Knobs &kn = Knobs{}, bool edges = false, bool exact_len = false, int over_lo = 0, int over_hi = 0, bool bytes = false) {
  // exact_len: every read read_len_base bases (no spread); over-long reads (one pair in twenty) of over_lo .. over_hi bases
  // (0: mrl + 5 .. mrl + 44)
  if (over_lo == 0) { over_lo = mrl + 5; over_hi = mrl + 44; }
  std::mt19937 g((unsigned)seed);
  RunStats rs;
  // ---- reference: two sequences, a 300 bp family with many copies, a 2 kb segmental repeat, an N run
  std::vector<std::string> seq = {std::string(edges ? 50000 : fam_copies > 200 ? 260000 : 70000, 'A'), std::string(edges ? 20000 : fam_copies > 200 ? 200000 : 50000, 'A')};
  for (auto &s : seq) for (auto &c : s) c = "ACGT"[g() %% 4];
  std::string fam(300, 'A'); for (auto &c : fam) c = "ACGT"[g() %% 4];
  for (int q = 0; q < fam_copies; ++q) { std::string f2 = fam; for (int x = 0; x < (int)(g() %% 4); ++x) f2[g() %% 300] = "ACGT"[g() %% 4]; std::string &s = seq[g() %% 2]; s.replace(500 + g() %% (s.size() - 1500), 300, f2); }
  std::string seg(2000, 'A'); for (auto &c : seg) c = "ACGT"[g() %% 4];
  for (int q = 0; q < 12; ++q) { std::string &s = seq[g() %% 2]; s.replace(1000 + g() %% (s.size() - 4000), 2000, seg); }
  seq[0].replace(30000, 80, std::string(80, 'N'));
  for (int q = 0; q < 3000; ++q) { std::string &s = seq[g() %% 2]; const size_t at = g() %% s.size(); s[at] = (char)tolower(s[at]); }
  if (bytes) {   // beyond upper-case ACGTN: soft-masked stretches of 50 to 2,000 bases over about 40 %%, IUPAC codes in both cases, bytes 0x80-0xFF
    for (auto &s : seq) {
      for (size_t masked = 0; masked < s.size() * 2 / 5;) {
        const size_t ln = 50 + g() %% 1951, at = g() %% (s.size() - ln);
        for (size_t i = at; i < at + ln; ++i) if (s[i] >= 'A' && s[i] <= 'Z') s[i] = (char)(s[i] + 32);
        masked += ln;
      }
      for (size_t q = 0; q < s.size() / 400; ++q) s[g() %% s.size()] = "RYKMSWBDHVrykmswbdhv"[g() %% 20];
      for (size_t q = 0; q < s.size() / 120; ++q) s[g() %% s.size()] = (char)(0x80 + g() %% 128);
    }
  }
  if (edges) {   // then many short sequences, as in a scaffold-level assembly: shorter than k + w - 1 (no minimizer), around L + 2e
                 // (no valid candidate), around a fragment, and a spread up to 3 kbp
    for (int len : {20, 30, 45, 60, 76, 80, 85, 90, 99, 100, 101, 110, 120, 136, 150, 180, 250, 400, 700, 1200, 3000}) seq.emplace_back((size_t)len, 'A');
    for (int q = 0; q < 24; ++q) seq.emplace_back((size_t)(64 + 64 * (g() %% 46)), 'A');
    for (size_t i = 2; i < seq.size(); ++i) {
      for (auto &c : seq[i]) c = "ACGT"[g() %% 4];
      // copies of the repeat family at both ends of the longer ones: with -f low enough a mate inside a copy has no candidates of
      // its own and is found by the mate-guided lookup around its partner, near the sequence's start or end
      if (seq[i].size() >= 1000) { seq[i].replace(0, 300, fam); seq[i].replace(seq[i].size() - 300, 300, fam); }
    }
  }
  const u32 n_seq = (u32)seq.size();
  std::string concat;
  std::vector<u64> offs{0};
  std::vector<std::string> nm;
  std::vector<const char *> names;
  for (u32 q = 0; q < n_seq; ++q) { concat += seq[q]; offs.push_back(concat.size()); nm.push_back("seq" + std::to_string(q)); }
  for (auto &s : nm) names.push_back(s.c_str());
  orc_reference *oref = orc_reference_from_memory(n_seq, concat.data(), (const uint64_t *)offs.data(), names.data());
  orc_index *oix = orc_index_build(oref, K, W);
  // ---- reads
  std::string s1, s2;
  std::vector<u32> o1{0}, o2{0};
  for (int p = 0; p < n_pairs; ++p) {
    const int kind = (int)(g() %% 20);
    int L1 = read_len_base + (int)(g() %% 11) - 5, L2 = read_len_base + (int)(g() %% 11) - 5;
    if (exact_len) L1 = L2 = read_len_base;
    if (kind == 0) L1 = over_lo + (int)(g() %% (unsigned)(over_hi - over_lo + 1));   // longer than the first tier allows
    if (kind == 1) L2 = 20;                                           // below the length filter
    const std::string &rsq = seq[g() %% (edges ? n_seq : 2)];
    int frag = std::max(L1, L2) + (int)(g() %% 350);
    size_t at;
    if (!edges) at = 200 + g() %% (rsq.size() - frag - 400);
    else {   // a third start within 40 bp of the sequence's start, a third end within 40 bp of its end, a third anywhere
      const int longest = std::max(L1, L2), size = (int)rsq.size();
      if (frag > size) frag = size > longest ? longest + (int)(g() %% (unsigned)(size - longest + 1)) : size;
      const size_t room = rsq.size() - (size_t)frag, near = std::min<size_t>(room, 40) + 1;
      const int where = (int)(g() %% 3);
      const size_t d = g() %% (1 + g() %% near);   // (more often the nearer)
      at = where == 0 ? d : where == 1 ? room - d : g() %% (room + 1);
    }
    std::string F = rsq.substr(at, (size_t)frag);
    while ((int)F.size() < std::max(L1, L2)) F += "ACGT"[g() %% 4];   // a sequence shorter than the reads: they run off its end
    frag = (int)F.size();
    if (kind == 2 || (fam_copies > 200 && kind %% 2 == 0)) { F = fam + std::string(rsq, at, (size_t)std::max(0, frag - 300)); F.resize((size_t)frag, 'A'); }   // inside the repeat family
    if (kind == 3) for (auto &c : F) c = "ACGT"[g() %% 4];                                                             // junk
    std::string a = F.substr(0, (size_t)L1), b = revc(F.substr((size_t)(frag - L2), (size_t)L2));
    if (mode == MODE_ATAC && g() %% 3 == 0 && std::min(L1, L2) > 40) {   // a fragment shorter than the reads: both mates run through into adapter sequence
      const int fl = 35 + (int)(g() %% (unsigned)(std::min(L1, L2) - 36));
      const std::string f2 = F.substr(0, (size_t)fl);
      a = f2 + std::string("CTGTCTCTTATACACATCTCCGAGCCCACGAGACAGGTTCAGAGTTCTACAGTCCGACGATCCTGTCTCTTATACACATCTCCGAGCCCACGAGAC").substr(0, (size_t)(L1 - fl));
      b = revc(f2) + std::string("CTGTCTCTTATACACATCTGACGCTGCCGACGAAGGTTCAGAGTTCTACAGTCCGACGATCACTGTCTCTTATACACATCTGACGCTGCCGACGA").substr(0, (size_t)(L2 - fl));
    }
    if (mode == MODE_HIC && g() %% 3 == 0 && L1 > 60) {    // a chimeric read: the far side of a ligation junction comes from another locus
      const std::string &r2 = seq[g() %% 2];
      const int cut = 30 + (int)(g() %% (unsigned)(L1 - 45));
      a = a.substr(0, (size_t)cut) + r2.substr(300 + g() %% (r2.size() - 1000), (size_t)(L1 - cut));
    }
    if (g() & 1) std::swap(a, b);
    for (std::string *r : {&a, &b}) {
      const int deco = bytes ? (int)(g() %% 7) : -1;   // (bytes) one read in seven keeps the reference high bytes it was copied from, 32 lower
      for (auto &c : *r) {
        if (c >= 'a' && c <= 'z') c = (char)(c - 32);
        // what a sequencer reads where the reference has no base; or (decoration 6) a high byte copied 32 lower, opposite its reference byte
        if (bytes && !strchr("ACGTN", c)) c = deco == 6 && (u8)c >= 0x80 ? (char)((u8)c - 32) : "ACGT"[g() %% 4];
      }
      const int ne = (int)(g() %% 4);
      for (int x = 0; x < ne; ++x) {
        const int k = (int)(g() %% 5), p2 = (int)(g() %% r->size());
        if (k < 3) (*r)[p2] = "ACGT"[g() %% 4];
        else if (k == 3) { r->erase((size_t)p2, 1); r->push_back("ACGT"[g() %% 4]); }
        else (*r)[p2] = 'N';
      }
    }
    if ((int)a.size() != L1) a.resize((size_t)L1, 'A');
    if ((int)b.size() != L2) b.resize((size_t)L2, 'A');
    for (std::string *r : {&a, &b}) {   // per read: none, wholly lower case, lower-case runs, 'n', '.', IUPAC codes (high bytes: above)
      if (!bytes) break;
      const int deco = (int)(g() %% 6), nr = (int)r->size();
      auto lower = [](char &c) { if (c >= 'A' && c <= 'Z') c = (char)(c + 32); };
      if (deco == 1) for (auto &c : *r) lower(c);
      if (deco == 2) for (int q = 1 + (int)(g() %% 3); q > 0; --q) { const int ln = 5 + (int)(g() %% 36), at = (int)(g() %% (unsigned)std::max(1, nr - ln)); for (int i = at; i < std::min(nr, at + ln); ++i) lower((*r)[i]); }
      if (deco >= 3) for (int q = 1 + (int)(g() %% 3); q > 0; --q) (*r)[g() %% nr] = deco == 3 ? 'n' : deco == 4 ? '.' : "RYKMSWBDHVrykmswbdhv"[g() %% 20];
    }
    s1 += a; o1.push_back((u32)s1.size()); s2 += b; o2.push_back((u32)s2.size());
  }
  const int n = n_pairs;
  // ---- oracle
  orc_params op; orc_default_params(&op); orc_apply_preset(&op, mode == MODE_ATAC ? "atac" : mode == MODE_HIC ? "hic" : "chip");
  op.max_num_best_mappings = max_best;
  if (kn.e >= 0) op.error_threshold = kn.e;
  if (kn.min_seeds >= 0) op.min_num_seeds = kn.min_seeds;
  if (kn.f0 >= 0) op.max_seed_freq0 = kn.f0;
  if (kn.f1 >= 0) op.max_seed_freq1 = kn.f1;
  if (kn.drop_rep >= 0) op.drop_repetitive_reads = kn.drop_rep;
  if (kn.min_read_len >= 0) op.min_read_length = kn.min_read_len;
  const bool is_se = mode == MODE_SE || mode == MODE_SAM_SE, is_sam = mode == MODE_SAM || mode == MODE_SAM_SE;
  op.single_end = is_se;
  orc_mapper *om = orc_mapper_create(&op, oix, oref);
  std::vector<orc_pe_record> want((size_t)n * max_best + 8);
  const u32 first_read_id = 5000;
  std::vector<orc_sam_record> want_sam;
  long n_want_sam = 0;
  if (is_sam) { want_sam.resize((size_t)n * max_best + 8); n_want_sam = (long)orc_map_sam_cores(om, (u32)n, s1.data(), o1.data(), is_se ? nullptr : s2.data(), is_se ? nullptr : o2.data(), first_read_id, want_sam.data(), (long)want_sam.size()); }
  std::vector<orc_pair_trace> trace((size_t)n);
  const long n_want = is_sam ? 0 : mode == MODE_SE ? (long)orc_map_reads_se(om, (u32)n, s1.data(), o1.data(), first_read_id, want.data(), (long)want.size(), 1)
                                      : (long)orc_map_pairs(om, (u32)n, s1.data(), o1.data(), s2.data(), o2.data(), first_read_id, want.data(), (long)want.size(), trace.data());
  if (bytes) {
    auto tally_lower = [&](u32 read_id, int strand) {
      const u32 p = read_id - first_read_id;
      bool lc = false;
      for (u32 i = o1[p]; i < o1[p + 1]; ++i) lc |= s1[i] >= 'a' && s1[i] <= 'z';
      if (lc) ++(strand ? rs.lower_s1 : rs.lower_s0);
    };
    if (is_sam) for (long i = 0; i < n_want_sam; ++i) tally_lower(want_sam[i].read_id, want_sam[i].strand[0]);
    else if (mode == MODE_HIC) for (long i = 0; i < n_want; ++i) tally_lower(((const orc_pairs_record *)want.data())[i].read_id, ((const orc_pairs_record *)want.data())[i].strand1);
    else for (long i = 0; i < n_want; ++i) tally_lower(want[i].read_id, want[i].direction);
  }
  if (edges) {   // what the oracle mapped at the edges: [st, en) on rid, with the mate-guided lookup run or not
    const u32 L = (u32)read_len_base, e = (u32)op.error_threshold, range = (u32)op.max_insert_size;
    auto tally_edges = [&](u32 rid, u32 st, u32 en, bool looked_up) {
      const u32 len = (u32)seq[rid].size();
      if (rid > 0 && st < L + e) ++rs.edge_start;
      if (en + e + 1 >= len) ++rs.edge_end;
      if (len < 2 * L) ++rs.short_seq;
      if (looked_up && rid > 0 && en <= 2 * range) ++rs.lookup_at_start;
    };
    if (is_sam) {
      for (long i = 0; i < n_want_sam; ++i) {
        const orc_sam_record &w = want_sam[i];
        tally_edges(w.rid, is_se ? w.pos[0] : std::min(w.pos[0], w.pos[1]), (is_se ? w.end[0] : std::max(w.end[0], w.end[1])) + 1, false);
      }
    } else if (mode == MODE_HIC) {
      for (long i = 0; i < n_want; ++i) {
        const orc_pairs_record &w = ((const orc_pairs_record *)want.data())[i];
        tally_edges(w.rid1, w.pos1, w.pos1 + 1, false);
        tally_edges(w.rid2, w.pos2, w.pos2 + 1, false);
      }
    } else {
      for (long i = 0; i < n_want; ++i) {   // a record for a pair with a mate without candidates of its own: the lookup found it
        const orc_pair_trace &t = trace[want[i].read_id - first_read_id];
        const bool looked_up = mode != MODE_SE && (t.supplement_result != 0 || t.n_pos_candidates_gen[0] + t.n_neg_candidates_gen[0] == 0 ||
                                                   t.n_pos_candidates_gen[1] + t.n_neg_candidates_gen[1] == 0);
        tally_edges(want[i].rid, want[i].fragment_start, want[i].fragment_start + want[i].fragment_length, looked_up);
      }
    }
  }
  // ---- device objects
  const DevParams P = dev_params(op, K, W);
  const uint32_t *kf; const uint64_t *kk, *kv, *kocc; uint32_t n_occ = 0;
  const uint32_t nb = orc_index_arrays(oix, &kf, &kk, &kv, &kocc, &n_occ);
  // the library's table: 16-byte slots {hash << 1 | singleton, value}, slot = (hash * phi64) >> shift, linear probing, load <= 0.5
  u64 n_keys = 0;
  for (uint32_t i = 0; i < nb; ++i) if (((kf[i >> 4] >> ((i & 0xfU) << 1)) & 3) == 0) ++n_keys;
  u64 n_slots_t = 16; while (n_slots_t < 2 * n_keys) n_slots_t <<= 1;
  int lg = 0; while ((1ull << lg) < n_slots_t) ++lg;
  std::vector<ulonglong2> slots((size_t)n_slots_t, ulonglong2{CMX_EMPTY_KEY, 0});
  for (uint32_t i = 0; i < nb; ++i) {
    if (((kf[i >> 4] >> ((i & 0xfU) << 1)) & 3) != 0) continue;
    u64 sidx = ((u64)(kk[i] >> 1) * 0x9E3779B97F4A7C15ull) >> (64 - lg);
    while (slots[sidx].x != CMX_EMPTY_KEY) sidx = (sidx + 1) & (n_slots_t - 1);
    slots[sidx] = ulonglong2{(u64)kk[i], (u64)kv[i]};
  }
  DevIndex ix{};
  ix.slots = slots.data(); ix.n_slots_mask = n_slots_t - 1; ix.shift = 64 - lg; ix.occ = (const u64 *)kocc; ix.n_occ = n_occ; ix.k = K; ix.w = W;
  // the library's reference layout, in an allocation of exactly its size (AddressSanitizer sees a read past the last padding)
  std::vector<u64> roff(n_seq);
  std::vector<u32> rlen(n_seq);
  std::vector<u8> refmem(ref_layout(n_seq, offs.data(), roff.data()), 0);
  for (u32 q = 0; q < n_seq; ++q) { rlen[q] = (u32)seq[q].size(); memcpy(refmem.data() + roff[q], seq[q].data(), rlen[q]); }
  DevRef R{refmem.data(), roff.data(), rlen.data(), n_seq};
  DevBatch B{};
  B.seq1 = (const u8 *)s1.data(); B.off1 = o1.data(); B.seq2 = (const u8 *)s2.data(); B.off2 = o2.data(); B.n_pairs = (u32)n; B.first_read_id = first_read_id;
  std::vector<double> il_(65536); std::vector<int> thr_(96);
  mapq_tables_fill(il_.data(), thr_.data());
  MapqTables T{il_.data(), thr_.data()};
  u32 mt_init[624];
  mt_init_fill(mt_init);
  // ---- run_lane's sequence
  Counters ctr{};
  std::vector<int> nbest((size_t)n, 0), sel((size_t)n * max_best, 0), out_n((size_t)n + 1, 0);
  std::vector<OutRecord> out_rec((size_t)n * max_best);
  std::vector<OutSam> out_sam(is_sam ? (size_t)n * max_best : 1);
  memset(out_sam.data(), 0, out_sam.size() * sizeof(OutSam));
  EmuLane x;
  for (int t = 0; t < N_TIERS; ++t) x.tiers[t].caps = caps3[t];
  const LaneArgs a{P, ix, R, B, T, mt_init, &ctr, x.cnt, nbest.data(), sel.data(), out_n.data(), is_sam ? (void *)out_sam.data() : (void *)out_rec.data(), is_sam, mrl};
  g_emu_leavable = true;
  {   // the tiles seed_front_kernel cannot stage (one grid over all pairs: tiles start at slot 0)
    const size_t tb = seed_front_tile_bytes(caps3[0].maxmm);
    for (int p0 = 0; p0 < n; p0 += SF_TILE)
      for (int m = 0; m < (is_se ? 1 : 2); ++m) {
        const std::string &sq = m == 0 ? s1 : s2;
        const std::vector<u32> &of = m == 0 ? o1 : o2;
        const u64 g0 = (u64)(sq.data() + of[(size_t)p0]), g1 = (u64)(sq.data() + of[(size_t)std::min(n, p0 + SF_TILE)]);
        rs.unstaged += g1 - (g0 & ~15ull) > tb;
      }
  }
  for (int p = 0; p < n; ++p) {   // mapped reads with 256 or more minimizers
    bool mapped = false;
    if (is_sam) { for (long i = 0; i < n_want_sam; ++i) mapped |= want_sam[i].read_id == first_read_id + (u32)p; }
    else if (mode == MODE_HIC) { for (long i = 0; i < n_want; ++i) mapped |= ((const orc_pairs_record *)want.data())[i].read_id == first_read_id + (u32)p; }
    else for (long i = 0; i < n_want; ++i) mapped |= want[i].read_id == first_read_id + (u32)p;
    if (!mapped) continue;
    for (int m = 0; m < (is_se ? 1 : 2); ++m) {
      std::vector<uint64_t> mh(8192), mhit(8192);
      const char *rd = m == 0 ? s1.data() + o1[p] : s2.data() + o2[p];
      const u32 len = m == 0 ? o1[p + 1] - o1[p] : o2[p + 1] - o2[p];
      rs.mm256 += orc_minimizers(rd, len, 0, K, W, mh.data(), mhit.data(), 8192) >= 256;
    }
  }
  // the front end: [adapter trimming] + length filter + minimizers + table probes over staged read tiles (seed_front_kernel, a
  // persistent grid: three CTAs here, so that every CTA walks several tiles through both stages of its double buffer)
  const Scratch S = lane_front(x, a, (u32)n, front_only ? 2 : 3);
  // cross-check of its records against the oracle's minimizers and khash lookups (what the kernel must have written)
  for (int slot = 0; slot < n; ++slot) {
    if (S.pmeta[slot].status != ST_OK) continue;
    for (int mate = 0; mate < (P.se ? 1 : 2); ++mate) {
      const ReadMeta &z = S.rmeta[2 * slot + mate];
      const char *rd = mate == 0 ? s1.data() + o1[slot] : s2.data() + o2[slot];
      std::vector<uint64_t> mh(4096), mhit(4096);
      const int nm = orc_minimizers(rd, (u32)z.len, 0, K, W, mh.data(), mhit.data(), 4096);
      bool ok = z.n_mm == nm && z.mm_done == 1;
      const size_t mb_ = mm_base(S, slot, mate);
      const int ms = mm_stride(S);
      for (int i = 0; ok && i < nm; ++i) {
        uint64_t key = 0, val = 0;
        const int found = orc_index_lookup(oix, mh[i], &key, &val);
        const u32 kind = found ? ((key & 1) ? 1u : 2u) : 0u;
        ok = S.mm_pos[mb_ + (size_t)i * ms] == (((u32)mhit[i] & 0x3FFFFFFFu) | (kind << 30)) && (!found || S.mm_val[mb_ + (size_t)i * ms] == val);
      }
      if (!ok) { if (rs.bad < 8) printf("FRONT END pair %%d mate %%d: n_mm %%d / %%d\n", slot, mate, z.n_mm, nm); ++rs.bad; }
    }
  }
  if (front_only) {   // (many tiles per CTA: both stages of the double buffer are refilled and both barrier phases flip)
    rs.pairs = n;
    rs.tier_pairs[0] = n;
    for (int slot = 0; slot < n; ++slot) rs.records += S.rmeta[2 * slot].n_mm + S.rmeta[2 * slot + 1].n_mm;
    g_emu_leavable = false;
    orc_mapper_free(om); orc_index_free(oix); orc_reference_free(oref);
    return rs;
  }
  const LaneTiers tiers = lane_tiers(x, a, S);
  for (int t = 0; t < tiers.used; ++t) rs.tier_pairs[t] = tiers.S[t].n_slots;
  rs.second_pass = x.cnt[3];   // (cluster_kernel's list counter: nothing after tier 0's clustering clears it)
  if (tiers.n_left > 0) { printf("pairs left after the last tier: %%d\n", tiers.n_left); ++rs.bad; }
  lane_emit(x, a, tiers, (u32)n);   // all pairs one reference batch
  g_emu_leavable = false;
  rs.max_smem = (long)x.max_smem; rs.cluster_launches = x.cluster_launches;
  // ---- compare, pair by pair
  if (is_sam) {
    static_assert(sizeof(OutSam) == sizeof(orc_sam_record), "SAM record layout");
    long si = 0;
    for (int p = 0; p < n; ++p) {
      long w0 = si;
      while (si < n_want_sam && want_sam[si].read_id == first_read_id + (u32)p) ++si;
      const int nw = (int)(si - w0);
      ++rs.pairs; rs.records += nw;
      bool ok = out_n[p] == nw;
      for (int r = 0; ok && r < nw; ++r) {
        const OutSam &a = out_sam[(size_t)p * max_best + r]; const orc_sam_record &b = want_sam[w0 + r];
        ok = a.read_id == b.read_id && a.rid == b.rid && a.pos[0] == b.pos[0] && a.end[0] == b.end[0] && a.strand[0] == b.strand[0] && a.n_cigar[0] == b.n_cigar[0] &&
             (is_se || (a.pos[1] == b.pos[1] && a.end[1] == b.end[1] && a.strand[1] == b.strand[1] && a.n_cigar[1] == b.n_cigar[1])) && a.mapq == b.mapq && a.is_unique == b.is_unique &&
             a.secondary == b.secondary &&
             a.overflow == b.overflow;
        for (int m = 0; ok && m < (is_se ? 1 : 2); ++m) for (int q = 0; ok && q < a.n_cigar[m]; ++q) ok = a.cigar[m][q] == b.cigar[m][q];
      }
      if (!ok) {
        if (rs.bad < 8) {
          printf("SAM PAIR %%d (seed %%d): records %%d / %%d", p, seed, out_n[p], nw);
          if (nw > 0 && out_n[p] > 0) { const OutSam &a = out_sam[(size_t)p * max_best]; const orc_sam_record &b = want_sam[w0];
            for (int m = 0; m < (is_se ? 1 : 2); ++m) printf("  mate %%d pos %%u/%%u end %%u/%%u strand %%u/%%u n_cigar %%u/%%u", m, a.pos[m], b.pos[m], a.end[m], b.end[m], a.strand[m], b.strand[m], a.n_cigar[m], b.n_cigar[m]);
            printf("  mapq %%u/%%u", a.mapq, b.mapq); }
          printf("\n");
        }
        ++rs.bad;
      }
    }
    if (si != n_want_sam) { printf("oracle SAM cores not consumed: %%ld of %%ld\n", si, n_want_sam); ++rs.bad; }
    orc_mapper_free(om); orc_index_free(oix); orc_reference_free(oref);
    return rs;
  }
  long wi = 0;
  for (int p = 0; p < n; ++p) {
    long w0 = wi;
    while (wi < n_want && want[wi].read_id == first_read_id + (u32)p) ++wi;
    const int nw = (int)(wi - w0);
    ++rs.pairs;
    rs.records += nw;
    bool ok = out_n[p] == nw;
    for (int r = 0; ok && r < nw; ++r) ok = memcmp(&out_rec[(size_t)p * max_best + r], &want[w0 + r], sizeof(OutRecord)) == 0;
    if (!ok) {
      if (rs.bad < 8) {
        printf("PAIR %%d (seed %%d): records %%d / %%d", p, seed, out_n[p], nw);
        if (nw > 0 && out_n[p] > 0) { const OutRecord &a = out_rec[(size_t)p * max_best]; const orc_pe_record &b = want[w0];
          printf("  rid %%u/%%u start %%u/%%u len %%u/%%u mapq %%u/%%u dir %%u/%%u uniq %%u/%%u", a.rid, b.rid, a.fragment_start, b.fragment_start, a.fragment_length, b.fragment_length, a.mapq, b.mapq, a.direction, b.direction, a.is_unique, b.is_unique); }
        printf("\n");
      }
      ++rs.bad;
    }
  }
  if (wi != n_want) { printf("oracle records not consumed: %%ld of %%ld\n", wi, n_want); ++rs.bad; }
  orc_mapper_free(om); orc_index_free(oix); orc_reference_free(oref);
  return rs;
}

int main(int argc, char **argv) {
  static_assert(sizeof(OutRecord) == sizeof(orc_pe_record) && sizeof(OutPairs) == sizeof(orc_pe_record), "record layouts");
  // the runs at the ends of reference sequences ("edges"), at the sizes a context grown beyond 160 bases takes ("grown"), else all others
  const bool want_edges = argc > 1 && !strcmp(argv[1], "edges"), want_grown = argc > 1 && !strcmp(argv[1], "grown"), want_bytes = argc > 1 && !strcmp(argv[1], "bytes");
  long bad = 0;
  const int mrl = 80;
  const Caps real[3] = {tier_caps(mrl, 0), tier_caps(mrl, 1), tier_caps(mrl, 2)};   // the library's tiers
  const Caps small[3] = {{mrl, 6, 2, 2}, {mrl * 2, 40, 6, 6}, {mrl * 4, 65536, 8192, 8192}};            // most pairs through the CTA kernels, some to the last tier
  const Caps real_long[3] = {tier_caps(150, 0), tier_caps(150, 1), tier_caps(150, 2)};
  const Caps small_long[3] = {{150, 6, 2, 2}, {300, 40, 6, 6}, {600, 65536, 8192, 8192}};
  const Caps small_256[3] = {{256, 6, 2, 2}, {512, 40, 6, 6}, {1024, 65536, 8192, 8192}};
  struct Case { const char *name; int mode, seed, n, max_best, len; const Caps *caps; int mrl; bool front_only = false; int k = 17, w = 7, fam_copies = 90; Knobs knobs = {}; bool edges = false;
                bool grown = false, exact = false; int over_lo = 0, over_hi = 0; bool bytes = false; };   // grown: caps nullptr = the library's tiers at mrl
  const Case cases[] = {
      {"real_tiers", MODE_CHIP, 3, 100, 1, 60, real, mrl},
      {"small_first_tier", MODE_CHIP, 4, 48, 3, 60, small, mrl},
      {"atac_trimming", MODE_ATAC, 5, 52, 1, 60, real, mrl},
      {"hic_split", MODE_HIC, 6, 44, 1, 120, real_long, 150},
      {"hic_split_cta", MODE_HIC, 7, 16, 1, 120, small_long, 150},
      {"single_end", MODE_SE, 8, 60, 2, 60, real, mrl},
      {"single_end_cta", MODE_SE, 9, 28, 1, 60, small, mrl},
      {"sam_cores", MODE_SAM, 10, 56, 2, 60, real, mrl},
      {"sam_cores_single_end", MODE_SAM_SE, 15, 40, 2, 60, real, mrl},
      {"heavy_repeats", MODE_CHIP, 14, 14, 2, 60, real, mrl, false, 17, 7, 420},       // a 420-copy family: thousands of hits, hundreds of candidates per read, up to the last tier
      {"front_end_only", MODE_CHIP, 11, 600, 1, 60, real, mrl, true},
      {"front_end_k21_w10", MODE_CHIP, 12, 200, 1, 60, real, mrl, true, 21, 10},     // the run-time scan (seed_front_kernel<false>)
      {"front_end_k16_w5", MODE_CHIP, 13, 200, 1, 60, real, mrl, true, 16, 5},       // even k: strand-symmetric k-mers
      // other index shapes, the whole pipeline: the run-time scan, k - 1 shifts of reverse-strand candidates, k + w - 1 overlaps
      // of repetitive seeds, the first cluster pass's rows by w.  For k > 22 the front end keeps every minimizer in the record arrays.
      {"k19_w10", MODE_CHIP, 16, 80, 1, 60, real, mrl, false, 19, 10},
      {"k19_w10_cta", MODE_CHIP, 17, 40, 2, 60, small, mrl, false, 19, 10},
      {"k23_w11", MODE_CHIP, 18, 80, 1, 60, real, mrl, false, 23, 11},
      {"k23_w11_cta", MODE_CHIP, 19, 40, 2, 60, small, mrl, false, 23, 11},
      {"k23_w11_single_end", MODE_SE, 20, 50, 2, 60, real, mrl, false, 23, 11},
      {"k23_w11_sam", MODE_SAM, 21, 40, 2, 60, real, mrl, false, 23, 11},
      {"k23_w11_hic", MODE_HIC, 22, 30, 1, 120, real_long, 150, false, 23, 11},
      {"k28_w20", MODE_CHIP, 23, 60, 1, 60, real, mrl, false, 28, 20},
      {"k16_w5", MODE_CHIP, 24, 60, 1, 60, real, mrl, false, 16, 5},
      // repetitive seeds at w > k: gaps between minimizers reach past k + 6, so the k + w - 1 overlap rule matters; MAPQ shows it
      // for uniquely mapped reads that run into a repeat copy
      {"k14_w30_repetitive", MODE_CHIP, 25, 100, 1, 120, real_long, 150, false, 14, 30, 90, Knobs{.f0 = 3, .f1 = 40}},
      {"k14_w30_repetitive_se", MODE_SE, 35, 100, 1, 120, real_long, 150, false, 14, 30, 90, Knobs{.f0 = 3, .f1 = 40}},
      // mapping knobs: error thresholds at both ends and across the 8 / 4 lane boundary, -n 8 through the CTA tiers, -s, -f low
      // enough for the second seeding round and repetitive-seed MAPQ, --drop-repetitive-reads, --min-read-length inside the read lengths
      {"e1", MODE_CHIP, 26, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.e = 1}},
      {"e7", MODE_CHIP, 27, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.e = 7}},
      {"e15", MODE_CHIP, 28, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.e = 15}},
      {"e15_cta", MODE_CHIP, 29, 30, 2, 60, small, mrl, false, 17, 7, 90, Knobs{.e = 15}},
      {"n8_cta", MODE_CHIP, 30, 40, 8, 60, small, mrl},
      {"s1", MODE_CHIP, 31, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.min_seeds = 1}},
      {"f3_40", MODE_CHIP, 32, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.f0 = 3, .f1 = 40}},
      {"drop20", MODE_CHIP, 33, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.drop_rep = 20}},
      {"min_read_length58", MODE_CHIP, 34, 60, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.min_read_len = 58}},
      // fragments at the ends of a 50 kbp, a 20 kbp and 45 short sequences (20 bp .. 3 kbp), both strands, every rid
      {"edges_chip", MODE_CHIP, 40, 400, 1, 60, real, mrl, false, 17, 7, 90, {}, true},
      {"edges_cta", MODE_CHIP, 41, 160, 2, 60, small, mrl, false, 17, 7, 90, {}, true},
      {"edges_e1", MODE_CHIP, 42, 160, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.e = 1}, true},
      {"edges_e15", MODE_CHIP, 43, 320, 1, 60, real, mrl, false, 17, 7, 90, Knobs{.e = 15}, true},
      {"edges_atac", MODE_ATAC, 44, 160, 1, 60, real, mrl, false, 17, 7, 90, {}, true},
      {"edges_hic", MODE_HIC, 45, 120, 1, 120, real_long, 150, false, 17, 7, 90, {}, true},
      {"edges_hic_cta", MODE_HIC, 46, 50, 1, 120, small_long, 150, false, 17, 7, 90, {}, true},
      {"edges_single_end", MODE_SE, 47, 200, 2, 60, real, mrl, false, 17, 7, 90, {}, true},
      {"edges_sam", MODE_SAM, 48, 160, 2, 60, real, mrl, false, 17, 7, 90, {}, true},
      {"edges_sam_single_end", MODE_SAM_SE, 49, 160, 2, 60, real, mrl, false, 17, 7, 90, {}, true},
      {"edges_f3_40", MODE_CHIP, 50, 300, 2, 60, real, mrl, false, 17, 7, 90, Knobs{.f0 = 3, .f1 = 40}, true},
      // contexts of 192 to 832 bases with the library's tiers: tier 0's hit rows 80 (192), 112 (256), 192 (from 448); two
      // cluster launches while the first-pass tile is shorter than hc (448, 704), one from 736; whole read-length tiles,
      // so that a tile with an over-long read is not staged (448 and up); at 832 the front end's tiles take 229,504 B and one
      // pair in twenty has a mate of 1,050 to 1,400 bases: the overflow tiers at maxmm 1,664 / 3,328, 256 or more minimizers
      {.name = "grown_chip192", .mode = MODE_CHIP, .seed = 60, .n = 96, .max_best = 1, .len = 186, .caps = nullptr, .mrl = 192, .fam_copies = 30, .grown = true},
      {.name = "grown_chip256", .mode = MODE_CHIP, .seed = 61, .n = 96, .max_best = 2, .len = 250, .caps = nullptr, .mrl = 256, .fam_copies = 30, .grown = true},
      {.name = "grown_chip448", .mode = MODE_CHIP, .seed = 62, .n = 80, .max_best = 1, .len = 448, .caps = nullptr, .mrl = 448, .fam_copies = 20, .grown = true, .exact = true},
      {.name = "grown_chip704", .mode = MODE_CHIP, .seed = 63, .n = 128, .max_best = 1, .len = 704, .caps = nullptr, .mrl = 704, .fam_copies = 10, .grown = true, .exact = true},
      {.name = "grown_chip736", .mode = MODE_CHIP, .seed = 64, .n = 80, .max_best = 1, .len = 736, .caps = nullptr, .mrl = 736, .fam_copies = 10, .grown = true, .exact = true},
      {.name = "grown_chip832", .mode = MODE_CHIP, .seed = 65, .n = 160, .max_best = 2, .len = 832, .caps = nullptr, .mrl = 832, .fam_copies = 20, .grown = true, .exact = true,
       .over_lo = 1050, .over_hi = 1400},
      // adapter trimming before the front end (prepped = 1), single-end, Hi-C split alignment in the thread and the CTA form
      {.name = "grown_atac256", .mode = MODE_ATAC, .seed = 66, .n = 80, .max_best = 1, .len = 250, .caps = nullptr, .mrl = 256, .fam_copies = 30, .grown = true},
      {.name = "grown_single_end320", .mode = MODE_SE, .seed = 67, .n = 96, .max_best = 2, .len = 314, .caps = nullptr, .mrl = 320, .fam_copies = 30, .grown = true},
      {.name = "grown_hic256", .mode = MODE_HIC, .seed = 68, .n = 64, .max_best = 1, .len = 250, .caps = nullptr, .mrl = 256, .fam_copies = 30, .grown = true},
      {.name = "grown_hic256_cta", .mode = MODE_HIC, .seed = 69, .n = 24, .max_best = 1, .len = 250, .caps = small_256, .mrl = 256, .fam_copies = 30, .grown = true},
      // --SAM above 160 bases: emit_sam_kernel<320> / emit_sam_se_kernel<320>, as lane_emit picks them (SAM reads stay within 320)
      {.name = "grown_sam256", .mode = MODE_SAM, .seed = 70, .n = 64, .max_best = 2, .len = 250, .caps = nullptr, .mrl = 256, .fam_copies = 30, .grown = true},
      {.name = "grown_sam_single_end320", .mode = MODE_SAM_SE, .seed = 71, .n = 64, .max_best = 2, .len = 300, .caps = nullptr, .mrl = 320, .fam_copies = 30, .grown = true,
       .over_lo = 306, .over_hi = 320},
      // k = 23: no key rows in the front end, the run-time scan, the first-pass tile by w = 11; then tiny first tiers: most
      // pairs through the CTA kernels at maxmm 512 / 1,024
      {.name = "grown_k23_w11_320", .mode = MODE_CHIP, .seed = 72, .n = 96, .max_best = 1, .len = 314, .caps = nullptr, .mrl = 320, .k = 23, .w = 11, .fam_copies = 30, .grown = true},
      {.name = "grown_small_tiers256", .mode = MODE_CHIP, .seed = 73, .n = 48, .max_best = 3, .len = 250, .caps = small_256, .mrl = 256, .fam_copies = 30, .grown = true},
      // reads and a reference beyond upper-case ACGTN: the raw-byte compares (Hamming shortcut of the traceback, adapter trimming,
      // Hi-C gap extension) and the case fold of every other step, in every mode, the CTA tiers and the 320-base SAM instance
      {.name = "bytes_chip", .mode = MODE_CHIP, .seed = 80, .n = 160, .max_best = 1, .len = 100, .caps = nullptr, .mrl = 128, .bytes = true},
      {.name = "bytes_chip_cta", .mode = MODE_CHIP, .seed = 81, .n = 64, .max_best = 2, .len = 60, .caps = small, .mrl = mrl, .bytes = true},
      {.name = "bytes_atac", .mode = MODE_ATAC, .seed = 82, .n = 160, .max_best = 1, .len = 100, .caps = nullptr, .mrl = 128, .bytes = true},
      {.name = "bytes_hic", .mode = MODE_HIC, .seed = 83, .n = 120, .max_best = 1, .len = 150, .caps = real_long, .mrl = 150, .bytes = true},
      {.name = "bytes_hic_cta", .mode = MODE_HIC, .seed = 84, .n = 40, .max_best = 1, .len = 120, .caps = small_long, .mrl = 150, .bytes = true},
      {.name = "bytes_single_end", .mode = MODE_SE, .seed = 85, .n = 160, .max_best = 2, .len = 100, .caps = nullptr, .mrl = 128, .bytes = true},
      {.name = "bytes_sam", .mode = MODE_SAM, .seed = 86, .n = 120, .max_best = 2, .len = 100, .caps = nullptr, .mrl = 128, .over_lo = 133, .over_hi = 160,
       .bytes = true},   // (SAM reads stay within the 160-base instance)
      {.name = "bytes_sam_single_end", .mode = MODE_SAM_SE, .seed = 87, .n = 120, .max_best = 2, .len = 100, .caps = nullptr, .mrl = 128, .over_lo = 133, .over_hi = 160,
       .bytes = true},   // (SAM reads stay within the 160-base instance)
      {.name = "bytes_sam256", .mode = MODE_SAM, .seed = 88, .n = 64, .max_best = 2, .len = 250, .caps = nullptr, .mrl = 256, .fam_copies = 30, .bytes = true},
  };
  const int seed_off = getenv("EMU_SEED_OFFSET") ? atoi(getenv("EMU_SEED_OFFSET")) : 0;   // other inputs of the same kinds (offline fuzzing)
  for (const Case &c : cases) {
    if (c.edges != want_edges || c.grown != want_grown || c.bytes != want_bytes) continue;
    Caps lib[3];
    for (int t = 0; t < 3; ++t) lib[t] = tier_caps(c.mrl, t);
    const RunStats r = run_case(c.mode, c.seed + seed_off, c.n, c.mrl, c.caps ? c.caps : lib, c.max_best, c.len, c.front_only, c.k, c.w, c.fam_copies, c.knobs, c.edges, c.exact,
                                c.over_lo, c.over_hi, c.bytes);
    printf("%%s: pairs=%%ld records=%%ld tier0=%%ld tier1=%%ld tier2=%%ld bad=%%ld edge_start=%%ld edge_end=%%ld short_seq=%%ld lookup_at_start=%%ld unstaged=%%ld second_pass=%%ld "
           "mm256=%%ld max_smem=%%ld cluster_launches=%%ld lower_s0=%%ld lower_s1=%%ld\n", c.name, r.pairs, r.records, r.tier_pairs[0], r.tier_pairs[1], r.tier_pairs[2], r.bad, r.edge_start, r.edge_end,
           r.short_seq, r.lookup_at_start, r.unstaged, r.second_pass, r.mm256, r.max_smem, r.cluster_launches, r.lower_s0, r.lower_s1);
    bad += r.bad;
    if (r.max_smem > 232448) { printf("%%s: a launch asks for %%ld B of dynamic shared memory, more than an H100 grants a CTA (232,448 B)\n", c.name, r.max_smem); ++bad; }
  }
  printf("total_bad=%%ld\n", bad);
  return bad != 0;
}
'''


def _run_cases(tmp_path, args=()):
    # CMX_EMU_SANITIZE=address | thread: the same run under AddressSanitizer (out-of-bounds accesses of reads, reference, table,
    # occurrence lists, shared memory) or ThreadSanitizer (the emulation's answer to racecheck: a missing __syncthreads between two
    # phases of a kernel is a data race between the OS threads that play the CUDA threads).  Minutes instead of seconds: on request.
    san = os.environ.get("CMX_EMU_SANITIZE", "")
    flags = ["-fsanitize=" + san, "-g", "-fno-omit-frame-pointer"] if san in ("address", "thread") else []
    exe = emu.build(tmp_path, emu.PIPELINE, MAIN % dict(orc_h=emu.ORACLE_H), flags=flags)
    if san == "address":
        os.environ["EMU_EXACT_SCRATCH"] = "1"
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0")
    out = subprocess.run([str(exe)] + list(args), capture_output=True, text=True, timeout=7200, env=env)
    assert out.returncode == 0 and "total_bad=0" in out.stdout, out.stdout[-3000:] + out.stderr[-800:]
    if san == "address":
        assert "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    if san == "thread":
        # two races are intended and harmless: a mate's thread flags its pair ST_OVERFLOW while the other mate's thread reads the status
        # (either order ends with the pair re-run in the next tier), and several threads clear cta_minimizers' fast-path flag (same value)
        reports = out.stderr.split("WARNING: ThreadSanitizer: data race")[1:]
        unexpected = [r for r in reports if not re.search(r"#0 (cluster_kernel|cta_minimizers)\(", r)]
        assert not unexpected, unexpected[0][:3000]
    return out


def test_device_pipeline_on_emulated_ctas_equals_the_oracle(tmp_path):
    out = _run_cases(tmp_path)
    got = {m.group(1): [int(x) for x in m.groups()[1:]] for m in re.finditer(r"(\w+): pairs=(\d+) records=(\d+) tier0=(\d+) tier1=(\d+) tier2=(\d+)", out.stdout)}
    assert got["real_tiers"][1] > 45 and got["real_tiers"][3] > 5, out.stdout                      # records; pairs that climbed to the second tier
    assert got["small_first_tier"][1] > 30 and got["small_first_tier"][3] > 20 and got["small_first_tier"][4] > 3, out.stdout   # CTA kernels, up to the last tier
    assert got["atac_trimming"][1] > 20 and got["hic_split"][1] > 18 and got["single_end"][1] > 25, out.stdout
    assert got["hic_split_cta"][3] > 3 and got["single_end_cta"][3] > 6 and got["sam_cores"][1] > 25 and got["sam_cores_single_end"][1] > 20 and got["heavy_repeats"][4] > 3 and got["front_end_only"][1] > 5000 and got["front_end_k21_w10"][1] > 800 and got["front_end_k16_w5"][1] > 1500, out.stdout
    # other index shapes and knobs: (records, pairs in the second tier, pairs in the last tier) at least
    floors = {"k19_w10": (50, 10, 0), "k19_w10_cta": (30, 15, 8), "k23_w11": (40, 12, 0), "k23_w11_cta": (25, 15, 8), "k23_w11_single_end": (35, 5, 0),
              "k23_w11_sam": (25, 5, 0), "k23_w11_hic": (18, 8, 0), "k28_w20": (15, 5, 0), "k16_w5": (40, 8, 0), "k14_w30_repetitive": (55, 0, 0), "k14_w30_repetitive_se": (50, 0, 0),
              "e1": (8, 12, 0), "e7": (30, 12, 0), "e15": (40, 12, 0), "e15_cta": (25, 15, 8), "n8_cta": (60, 15, 8), "s1": (40, 12, 0),
              "f3_40": (30, 4, 0), "drop20": (30, 10, 0), "min_read_length58": (18, 10, 0)}
    for name, (records, tier1, tier2) in floors.items():
        assert got[name][1] > records and got[name][3] >= tier1 and got[name][4] >= tier2, (name, out.stdout)


def test_device_pipeline_at_sequence_ends_equals_the_oracle(tmp_path):
    """Fragments that start or end within 40 bp of a sequence's ends, on every rid of a reference of one 50 kbp, one 20 kbp and
    45 short sequences (20 bp to 3 kbp, some shorter than k + w - 1, than L + 2e or than a fragment): candidate validity near both
    ends (valid_cand), the right-end clamp of the verification window, mate-guided lookups whose window begins below a rid's
    start, negative-strand candidates that wrap below position 0 — every mode, the CTA tiers included.  Each run must map enough at the edges to show it reached them."""
    out = _run_cases(tmp_path, ["edges"])
    got = {m.group(1): [int(x) for x in m.groups()[1:]] for m in
           re.finditer(r"(\w+): pairs=\d+ records=(\d+) tier0=\d+ tier1=(\d+) tier2=(\d+) bad=\d+ edge_start=(\d+) edge_end=(\d+) short_seq=(\d+) lookup_at_start=(\d+)", out.stdout)}
    # per run, at least: (records, pairs in the second tier, pairs in the last tier, records that start within L + e of a rid > 0's
    # start, records that end within e + 1 of a sequence's end, records on sequences shorter than 2L, pairs whose mate-guided lookup
    # window began below a rid > 0's start).  (Single-end, SAM and Hi-C runs have no mate-guided lookup; a Hi-C record holds 5' ends.)
    floors = {"edges_chip": (130, 90, 0, 30, 3, 3, 4), "edges_cta": (80, 90, 30, 12, 1, 0, 3), "edges_e1": (25, 40, 0, 7, 1, 2, 0),
              "edges_e15": (90, 70, 0, 9, 1, 0, 3), "edges_atac": (55, 35, 0, 12, 2, 2, 1), "edges_hic": (50, 35, 0, 9, 0, 1, 0),
              "edges_hic_cta": (15, 30, 8, 6, 0, 5, 0), "edges_single_end": (110, 30, 0, 18, 1, 7, 0), "edges_sam": (70, 30, 0, 12, 2, 1, 0),
              "edges_sam_single_end": (95, 35, 0, 25, 1, 8, 0), "edges_f3_40": (65, 8, 0, 24, 2, 4, 9)}
    for name, floor in floors.items():
        assert all(g >= f for g, f in zip(got[name], floor)), (name, out.stdout)
    # and over all runs
    total = [sum(got[name][i] for name in floors) for i in (4, 5, 6)]
    assert total[0] >= 15 and total[1] >= 35 and total[2] >= 22, (total, out.stdout)


def test_device_pipeline_at_grown_read_lengths_equals_the_oracle(tmp_path):
    """Contexts of 192 to 832 bases, with the tiers the library sizes for them (`tier_caps`): tier 0's hit rows of 80, 112
    and 192, one or two cluster_kernel passes, front-end tiles too long to stage (each thread then copies its own read), the
    overflow tiers at maxmm up to 3,328 with reads of 256 or more minimizers, adapter trimming, single-end, Hi-C in the thread
    and the CTA form, `--SAM` through the 320-base instances, k = 23 and tiny first tiers.  Each run must show that it reached
    what it is there for, and no launch may ask for more dynamic shared memory than an H100 grants one CTA (232,448 B)."""
    out = _run_cases(tmp_path, ["grown"])
    got = {m.group(1): [int(x) for x in m.groups()[1:]] for m in
           re.finditer(r"(\w+): pairs=\d+ records=(\d+) tier0=\d+ tier1=(\d+) tier2=(\d+) bad=\d+ edge_start=\d+ edge_end=\d+ short_seq=\d+ lookup_at_start=\d+ "
                       r"unstaged=(\d+) second_pass=(\d+) mm256=(\d+) max_smem=(\d+) cluster_launches=(\d+)", out.stdout)}
    # per run, at least: (records, pairs in the second tier, pairs in the last tier, unstaged front-end tiles, reads clustered by
    # cluster_kernel's second pass, reads of mapped pairs with 256 or more minimizers); then the number of cluster launches
    floors = {"grown_chip192": (60, 20, 0, 0, 1, 0, 2), "grown_chip256": (75, 20, 0, 0, 1, 0, 2), "grown_chip448": (45, 15, 1, 0, 1, 0, 2),
              "grown_chip704": (75, 30, 0, 1, 8, 0, 2), "grown_chip736": (50, 15, 0, 1, 0, 0, 1), "grown_chip832": (110, 80, 8, 1, 0, 2, 1),
              "grown_atac256": (40, 20, 0, 0, 0, 0, 2), "grown_single_end320": (75, 15, 0, 0, 1, 0, 2), "grown_hic256": (45, 15, 0, 0, 0, 0, 2),
              "grown_hic256_cta": (18, 18, 8, 0, 0, 0, 1), "grown_sam256": (50, 15, 0, 0, 0, 0, 2), "grown_sam_single_end320": (55, 15, 0, 0, 1, 0, 2),
              "grown_k23_w11_320": (60, 20, 0, 0, 1, 0, 2), "grown_small_tiers256": (40, 35, 20, 0, 0, 0, 1)}
    assert sorted(got) == sorted(floors), out.stdout
    for name, (*floor, launches) in floors.items():
        g = got[name]
        assert all(x >= f for x, f in zip(g[:6], floor)) and g[7] == launches and g[6] <= 232448, (name, out.stdout)
    # the front end's tiles at 832 bases: 4 x (64 x 832 + 32) + 16 x 128 x 8 bytes, the largest request of any launch there
    assert got["grown_chip832"][6] == 229504, out.stdout
    total = [sum(g[i] for g in got.values()) for i in (3, 4, 5)]
    assert total[0] >= 4 and total[1] >= 25 and total[2] >= 2, (total, out.stdout)


def test_device_pipeline_on_raw_bytes_equals_the_oracle(tmp_path):
    """A soft-masked reference (about 40 %) with IUPAC codes in both cases and bytes 0x80-0xFF; reads that are wholly or partly
    lower case, carry 'n', '.' or IUPAC codes, or a reference high byte copied 32 lower: the raw-byte compares of the Hamming
    shortcut in the traceback, adapter trimming and the Hi-C gap extension, and the case fold (base_code) everywhere else.
    Chip with the library's tiers and tiny ones, atac, Hi-C in the thread and the CTA form, single-end, `--SAM` paired and
    single-end, and 2x250 `--SAM` through the 320-base instance; each against the oracle pair by pair."""
    out = _run_cases(tmp_path, ["bytes"])
    got = {m.group(1): [int(x) for x in m.groups()[1:]] for m in
           re.finditer(r"(\w+): pairs=\d+ records=(\d+) tier0=\d+ tier1=(\d+) tier2=(\d+) .* lower_s0=(\d+) lower_s1=(\d+)", out.stdout)}
    # per run, at least: (records, pairs in the second tier, pairs in the last tier, records whose read 1 has a lower-case base with
    # strand field 0, the same with 1): about half of what the first run showed
    floors = {"bytes_chip": (59, 34, 0, 14, 22), "bytes_chip_cta": (25, 17, 13, 7, 7), "bytes_atac": (43, 35, 0, 16, 12), "bytes_hic": (53, 49, 0, 3, 31),
              "bytes_hic_cta": (17, 18, 12, 1, 10), "bytes_single_end": (82, 27, 0, 19, 35), "bytes_sam": (56, 29, 0, 13, 23),
              "bytes_sam_single_end": (60, 19, 0, 12, 22), "bytes_sam256": (17, 12, 0, 5, 6)}
    assert sorted(got) == sorted(floors), out.stdout
    for name, floor in floors.items():
        assert all(g >= f for g, f in zip(got[name], floor)), (name, out.stdout)
