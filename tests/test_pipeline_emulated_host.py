"""The whole device pipeline — seed_front -> cluster -> pair_candidates -> verify -> pairing (tier 0, thread kernels), prep ->
seed_cta -> pair_candidates_cta -> verify_cta -> pairing_cta (overflow tiers, one CTA per read / pair), overflow collection
between the tiers, select, emit (+ deferred tracebacks) / emit_cta — compiled from the UNCHANGED kernel sources
(device_common.cuh, minimizers.cuh, pipeline_kernels.cuh, seed_front.cuh, cta_pair_candidates.cuh, cta_verify_pairing.cuh, sam_kernels.cuh) and run on the host
emulation of CTAs (tests/cta_emu.h) with the launch sequence, grid / block sizes, shared-memory sizes and scratch layout of
the library's run_lane (the layout by the library's own `scratch_layout`), against the oracle's mapper (`orc_map_pairs`, pinned to the
reference binary by tests/test_oracle_golden.py): every pair's records, field by field.
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
read, the real capacities up to the last tier)."""
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
  std::vector<int> list;   // pair list of this tier (empty = identity)
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
template <typename F>
static void launch(int grid, int block, size_t smem_bytes, F body) {   // kernel<<<grid, block, smem>>>(...)
  g_smem.assign(smem_bytes / 8 + 2, 0xA5A5A5A5A5A5A5A5ull);
  g_dyn_smem = g_smem.data();
  emu_grid(grid, block, body);
}
static char comp(char c) { switch (c) { case 'A': case 'a': return 'T'; case 'C': case 'c': return 'G'; case 'G': case 'g': return 'C'; case 'T': case 't': return 'A'; default: return 'N'; } }
static std::string revc(const std::string &s) { std::string r(s.rbegin(), s.rend()); for (auto &c : r) c = comp(c); return r; }

struct RunStats { long pairs = 0, records = 0, tier_pairs[3] = {0, 0, 0}, bad = 0; };

enum { MODE_CHIP = 0, MODE_ATAC = 1, MODE_HIC = 2, MODE_SE = 3, MODE_SAM = 4, MODE_SAM_SE = 5 };
static RunStats run_case(int mode, int seed, int n_pairs, int mrl, const Caps *caps3, int max_best, int read_len_base, bool front_only = false, int K = 17, int W = 7, int fam_copies = 90) {
  std::mt19937 g((unsigned)seed);
  RunStats rs;
  // ---- reference: two sequences, a 300 bp family with many copies, a 2 kb segmental repeat, an N run
  std::string seq[2] = {std::string(fam_copies > 200 ? 260000 : 70000, 'A'), std::string(fam_copies > 200 ? 200000 : 50000, 'A')};
  for (auto &s : seq) for (auto &c : s) c = "ACGT"[g() %% 4];
  std::string fam(300, 'A'); for (auto &c : fam) c = "ACGT"[g() %% 4];
  for (int q = 0; q < fam_copies; ++q) { std::string f2 = fam; for (int x = 0; x < (int)(g() %% 4); ++x) f2[g() %% 300] = "ACGT"[g() %% 4]; std::string &s = seq[g() %% 2]; s.replace(500 + g() %% (s.size() - 1500), 300, f2); }
  std::string seg(2000, 'A'); for (auto &c : seg) c = "ACGT"[g() %% 4];
  for (int q = 0; q < 12; ++q) { std::string &s = seq[g() %% 2]; s.replace(1000 + g() %% (s.size() - 4000), 2000, seg); }
  seq[0].replace(30000, 80, std::string(80, 'N'));
  for (int q = 0; q < 3000; ++q) { std::string &s = seq[g() %% 2]; const size_t at = g() %% s.size(); s[at] = (char)tolower(s[at]); }
  std::string concat = seq[0] + seq[1];
  const uint64_t offs[3] = {0, seq[0].size(), seq[0].size() + seq[1].size()};
  const char *names[2] = {"chrA", "chrB"};
  orc_reference *oref = orc_reference_from_memory(2, concat.data(), offs, names);
  orc_index *oix = orc_index_build(oref, K, W);
  // ---- reads
  std::string s1, s2;
  std::vector<u32> o1{0}, o2{0};
  for (int p = 0; p < n_pairs; ++p) {
    const int kind = (int)(g() %% 20);
    int L1 = read_len_base + (int)(g() %% 11) - 5, L2 = read_len_base + (int)(g() %% 11) - 5;
    if (kind == 0) L1 = mrl + 5 + (int)(g() %% 40);                   // longer than the first tier allows
    if (kind == 1) L2 = 20;                                           // below the length filter
    const std::string &rsq = seq[g() %% 2];
    const int frag = std::max(L1, L2) + (int)(g() %% 350);
    size_t at = 200 + g() %% (rsq.size() - frag - 400);
    std::string F = rsq.substr(at, (size_t)frag);
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
      for (auto &c : *r) c = (char)toupper(c);
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
    s1 += a; o1.push_back((u32)s1.size()); s2 += b; o2.push_back((u32)s2.size());
  }
  const int n = n_pairs;
  // ---- oracle
  orc_params op; orc_default_params(&op); orc_apply_preset(&op, mode == MODE_ATAC ? "atac" : mode == MODE_HIC ? "hic" : "chip");
  op.max_num_best_mappings = max_best;
  const bool is_se = mode == MODE_SE || mode == MODE_SAM_SE, is_sam = mode == MODE_SAM || mode == MODE_SAM_SE;
  op.single_end = is_se;
  orc_mapper *om = orc_mapper_create(&op, oix, oref);
  std::vector<orc_pe_record> want((size_t)n * max_best + 8);
  const u32 first_read_id = 5000;
  std::vector<orc_sam_record> want_sam;
  long n_want_sam = 0;
  if (is_sam) { want_sam.resize((size_t)n * max_best + 8); n_want_sam = (long)orc_map_sam_cores(om, (u32)n, s1.data(), o1.data(), is_se ? nullptr : s2.data(), is_se ? nullptr : o2.data(), first_read_id, want_sam.data(), (long)want_sam.size()); }
  const long n_want = is_sam ? 0 : mode == MODE_SE ? (long)orc_map_reads_se(om, (u32)n, s1.data(), o1.data(), first_read_id, want.data(), (long)want.size(), 1)
                                      : (long)orc_map_pairs(om, (u32)n, s1.data(), o1.data(), s2.data(), o2.data(), first_read_id, want.data(), (long)want.size(), nullptr);
  // ---- device objects
  DevParams P{};
  P.e = op.error_threshold; P.min_seeds = op.min_num_seeds; P.f0 = op.max_seed_freq0; P.f1 = op.max_seed_freq1; P.max_best = max_best; P.max_insert = op.max_insert_size;
  P.min_read_len = op.min_read_length; P.drop_rep = op.drop_repetitive_reads; P.trim = op.trim_adapters; P.k = K; P.w = W; P.lanes = P.e < 8 ? 8 : 4; P.split = op.split_alignment;
  P.se = is_se;
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
  std::string refmem(64, '\0');
  u64 roff[2]; u32 rlen[2];
  for (int q = 0; q < 2; ++q) { roff[q] = refmem.size(); rlen[q] = (u32)seq[q].size(); refmem += seq[q]; refmem.append(64 + (64 - refmem.size() %% 64) %% 64, '\0'); }
  refmem.append(128, '\0');
  DevRef R{(const u8 *)refmem.data(), roff, rlen, 2};
  DevBatch B{};
  B.seq1 = (const u8 *)s1.data(); B.off1 = o1.data(); B.seq2 = (const u8 *)s2.data(); B.off2 = o2.data(); B.n_pairs = (u32)n; B.first_read_id = first_read_id;
  std::vector<double> il_(65536); std::vector<int> thr_(96);
  mapq_tables_fill(il_.data(), thr_.data());
  MapqTables T{il_.data(), thr_.data()};
  u32 mt_init[624];
  mt_init[0] = 11u;
  for (int i = 1; i < 624; ++i) mt_init[i] = 1812433253u * (mt_init[i - 1] ^ (mt_init[i - 1] >> 30)) + (u32)i;
  // ---- run_lane, tier by tier
  HostTier tiers[3];
  for (int t = 0; t < 3; ++t) tiers[t].caps = caps3[t];
  Counters ctr{};
  std::vector<int> nbest((size_t)n, 0), sel((size_t)n * max_best, 0), out_n((size_t)n + 1, 0);
  std::vector<OutRecord> out_rec((size_t)n * max_best);
  std::vector<OutSam> out_sam(is_sam ? (size_t)n * max_best : 1);
  memset(out_sam.data(), 0, out_sam.size() * sizeof(OutSam));
  int n_slots = n, tiers_used = 0;
  const int *pair_list = nullptr;
  const int TB = 128;
  g_emu_leavable = true;
  for (int t = 0; t < 3 && n_slots > 0; ++t) {
    HostTier &tier = tiers[t];
    tier_prepare_host(tier, n_slots, pair_list, t == 0);
    const Scratch S = tier.view;
    rs.tier_pairs[t] = n_slots;
    if (t == 0) {
      // the front end: [adapter trimming] + length filter + minimizers + table probes over staged read tiles (seed_front_kernel, a
      // persistent grid: three CTAs here, so that every CTA walks several tiles through both stages of its double buffer)
      if (P.trim) launch((n_slots + TB - 1) / TB, TB, 0, [&]() { prep_kernel(P, B, S); });
      {
        const int tiles = (n_slots + SF_TILE - 1) / SF_TILE;
        launch(front_only ? 2 : std::min(tiles, 3), SF_NT, seed_front_smem_bytes(S.caps.maxmm) + 16, [&]() { if (K == 17 && W == 7) seed_front_kernel<true>(P, ix, B, S, &ctr, P.trim ? 1 : 0, 0, n_slots); else seed_front_kernel<false>(P, ix, B, S, &ctr, P.trim ? 1 : 0, 0, n_slots); });
      }
      // cross-check of its records against the oracle's minimizers and khash lookups (what the kernel must have written)
      for (int slot = 0; slot < n_slots; ++slot) {
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
        rs.pairs = n_slots;
        for (int slot = 0; slot < n_slots; ++slot) rs.records += S.rmeta[2 * slot].n_mm + S.rmeta[2 * slot + 1].n_mm;
        g_emu_leavable = false;
        orc_mapper_free(om); orc_index_free(oix); orc_reference_free(oref);
        return rs;
      }
      std::vector<int> vlist((size_t)2 * n_slots + 8), rlist((size_t)n_slots + 8);
      int d_count[4] = {0, 0, 0, 0};
      int rows0 = (2 * mrl / (7 + 1) + 15) / 16 * 16;
      rows0 = std::max(16, std::min(rows0, S.caps.hc));
      launch((2 * n_slots + CLUSTER_NT - 1) / CLUSTER_NT, CLUSTER_NT, (size_t)rows0 * CLUSTER_NT * 8, [&]() { cluster_kernel(P, ix, S, &ctr, 0, rows0, vlist.data(), &d_count[3]); });
      if (rows0 < S.caps.hc)
        launch((2 * n_slots + CLUSTER_NT - 1) / CLUSTER_NT, CLUSTER_NT, (size_t)S.caps.hc * CLUSTER_NT * 8, [&]() { cluster_kernel(P, ix, S, &ctr, 1, S.caps.hc, vlist.data(), &d_count[3]); });
      launch((n_slots + TB - 1) / TB, TB, 0, [&]() { pair_candidates_kernel(P, ix, S, &ctr, 0, rlist.data(), &d_count[1]); });
      launch((n_slots + 63) / 64, 64, 0, [&]() { pair_candidates_kernel(P, ix, S, &ctr, 1, rlist.data(), &d_count[1]); });
      if (P.split) launch((2 * n_slots + TB - 1) / TB, TB, 0, [&]() { verify_split_kernel(P, R, B, S, &ctr); });
      else {
        launch((2 * n_slots + TB - 1) / TB, TB, 0, [&]() { verify_kernel(P, R, B, S, &ctr, 0, vlist.data(), &d_count[2]); });
        launch((2 * n_slots + 63) / 64, 64, (size_t)2 * S.caps.maxmm * 64, [&]() { verify_kernel(P, R, B, S, &ctr, 1, vlist.data(), &d_count[2]); });
      }
      if (P.split) launch((n_slots + TB - 1) / TB, TB, 0, [&]() { pairing_split_kernel(P, S, nbest.data()); });
      else launch((n_slots + TB - 1) / TB, TB, 0, [&]() { pairing_kernel(P, S, nbest.data()); });
    } else {
      auto cap_of = [](int c_) { int c = 1; while (c < c_) c <<= 1; return std::min(c, CTA_SORT_SMEM_MAX); };
      const int c_seed = cap_of(2 * tier.caps.hc), c_pc = cap_of(tier.caps.hc), c_ver = cap_of(tier.caps.cc), c_pair = cap_of(tier.caps.mc);
      launch((n_slots + TB - 1) / TB, TB, 0, [&]() { prep_kernel(P, B, S); });
      launch(2 * n_slots, CTA_NT, (size_t)c_seed * 11 + (size_t)(tier.caps.maxmm + 1) * 12 + 16, [&]() { seed_cta_kernel(P, ix, B, S, tiers[0].view, &ctr, c_seed); });
      const int lcap = std::min(tier.caps.cc, 512), fcap = 2 * tier.caps.cc;
      const size_t pc_smem = pair_candidates_cta_smem(c_pc, lcap, tier.caps.maxmm, fcap);
      const int pc_nt = pc_smem > 64 * 1024 ? PC_CTA_NT_MAX : CTA_NT;
      launch(n_slots, pc_nt, pc_smem, [&]() { pair_candidates_cta_kernel(P, ix, S, &ctr, c_pc, lcap, fcap, nullptr, nullptr); });
      if (P.split) launch(2 * n_slots, CTA_NT, (size_t)c_ver * 9, [&]() { verify_split_cta_kernel(P, R, B, S, &ctr, c_ver); });
      else launch(2 * n_slots, tier.caps.cc > 1024 ? VERIFY_NT_MAX : CTA_NT, (size_t)c_ver * 9 + 2 * (size_t)tier.caps.maxmm + 16, [&]() { verify_cta_kernel(P, R, B, S, &ctr, c_ver); });
      if (P.split) launch((n_slots + TB - 1) / TB, TB, 0, [&]() { pairing_split_kernel(P, S, nbest.data()); });
      else launch(n_slots, CTA_NT, (size_t)c_pair * 10, [&]() { pairing_cta_kernel(P, S, nbest.data(), c_pair); });
    }
    std::vector<int> ovf((size_t)n_slots + 8);
    int n_ovf = 0;
    launch((n_slots + 255) / 256, 256, 0, [&]() { collect_overflow_kernel(S, ovf.data(), &n_ovf); });
    tiers_used = t + 1;
    if (n_ovf > 0 && t + 1 < 3) {
      ovf.resize((size_t)n_ovf);
      std::sort(ovf.begin(), ovf.end());
      tiers[t + 1].list = ovf;
      pair_list = tiers[t + 1].list.data();
    } else if (n_ovf > 0) { printf("pairs left after the last tier: %%d\n", n_ovf); ++rs.bad; }
    n_slots = n_ovf;
  }
  // one reference batch = all pairs here: taskloop chunks of n / (n / 5000) ...: a single chunk for n < 10000
  int chunks[2] = {0, n};
  launch(1, 128, 0, [&]() { select_kernel(P, 1, chunks, nbest.data(), sel.data(), mt_init); });
  for (int t = tiers_used - 1; t >= 0; --t) {
    const Scratch S = tiers[t].view;
    if (mode == MODE_SAM_SE) launch((S.n_slots + TB - 1) / TB, TB, 0, [&]() { emit_sam_se_kernel(P, R, B, T, S, sel.data(), out_sam.data(), out_n.data(), &ctr); });
    else if (mode == MODE_SAM) launch((S.n_slots + TB - 1) / TB, TB, 0, [&]() { emit_sam_kernel(P, R, B, T, S, sel.data(), out_sam.data(), out_n.data(), &ctr); });
    else if (P.split) launch((S.n_slots + TB - 1) / TB, TB, 0, [&]() { emit_split_kernel(P, R, B, T, S, sel.data(), (OutPairs *)out_rec.data(), out_n.data(), &ctr); });
    else if (P.se) launch((S.n_slots + TB - 1) / TB, TB, 0, [&]() { emit_se_kernel(P, R, B, T, S, sel.data(), out_rec.data(), out_n.data(), &ctr); });
    else if (t > 0) launch(S.n_slots, CTA_NT, 0, [&]() { emit_cta_kernel(P, R, B, T, S, sel.data(), out_rec.data(), out_n.data(), &ctr); });
    else {
      std::vector<int4> emit_list((size_t)S.n_slots * max_best + 8);
      int dp_count = 0;
      launch((S.n_slots + TB - 1) / TB, TB, 0, [&]() { emit_kernel(P, R, B, T, S, sel.data(), out_rec.data(), out_n.data(), &ctr, emit_list.data(), &dp_count); });
      launch((int)(((size_t)S.n_slots * max_best + TB - 1) / TB), TB, 0, [&]() { emit_dp_kernel(P, R, B, T, S, out_rec.data(), emit_list.data(), &dp_count); });
    }
  }
  g_emu_leavable = false;
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
      if (!ok) { if (rs.bad < 8) printf("SAM PAIR %%d (seed %%d): records %%d / %%d\n", p, seed, out_n[p], nw); ++rs.bad; }
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

int main() {
  static_assert(sizeof(OutRecord) == sizeof(orc_pe_record) && sizeof(OutPairs) == sizeof(orc_pe_record), "record layouts");
  long bad = 0;
  const int mrl = 80;
  const Caps real[3] = {{mrl, 64, 32, 32}, {mrl * 2, 1024, 256, 256}, {mrl * 4, 65536, 8192, 8192}};   // the library's tiers
  const Caps small[3] = {{mrl, 6, 2, 2}, {mrl * 2, 40, 6, 6}, {mrl * 4, 65536, 8192, 8192}};            // most pairs through the CTA kernels, some to the last tier
  const Caps real_long[3] = {{150, 64, 32, 32}, {300, 1024, 256, 256}, {600, 65536, 8192, 8192}};
  const Caps small_long[3] = {{150, 6, 2, 2}, {300, 40, 6, 6}, {600, 65536, 8192, 8192}};
  struct Case { const char *name; int mode, seed, n, max_best, len; const Caps *caps; int mrl; bool front_only = false; int k = 17, w = 7, fam_copies = 90; };
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
  };
  const int seed_off = getenv("EMU_SEED_OFFSET") ? atoi(getenv("EMU_SEED_OFFSET")) : 0;   // other inputs of the same kinds (offline fuzzing)
  for (const Case &c : cases) {
    const RunStats r = run_case(c.mode, c.seed + seed_off, c.n, c.mrl, c.caps, c.max_best, c.len, c.front_only, c.k, c.w, c.fam_copies);
    printf("%%s: pairs=%%ld records=%%ld tier0=%%ld tier1=%%ld tier2=%%ld bad=%%ld\n", c.name, r.pairs, r.records, r.tier_pairs[0], r.tier_pairs[1], r.tier_pairs[2], r.bad);
    bad += r.bad;
  }
  printf("total_bad=%%ld\n", bad);
  return bad != 0;
}
'''


def test_device_pipeline_on_emulated_ctas_equals_the_oracle(tmp_path):
    # CMX_EMU_SANITIZE=address | thread: the same run under AddressSanitizer (out-of-bounds accesses of reads, reference, table,
    # occurrence lists, shared memory) or ThreadSanitizer (the emulation's answer to racecheck: a missing __syncthreads between two
    # phases of a kernel is a data race between the OS threads that play the CUDA threads).  Minutes instead of seconds: on request.
    san = os.environ.get("CMX_EMU_SANITIZE", "")
    flags = ["-fsanitize=" + san, "-g", "-fno-omit-frame-pointer"] if san in ("address", "thread") else []
    exe = emu.build(tmp_path, emu.PIPELINE, MAIN % dict(orc_h=emu.ORACLE_H), flags=flags)
    if san == "address":
        os.environ["EMU_EXACT_SCRATCH"] = "1"
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0")
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=7200, env=env)
    assert out.returncode == 0 and "total_bad=0" in out.stdout, out.stdout[-3000:] + out.stderr[-800:]
    if san == "address":
        assert "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    if san == "thread":
        # two races are intended and harmless: a mate's thread flags its pair ST_OVERFLOW while the other mate's thread reads the status
        # (either order ends with the pair re-run in the next tier), and several threads clear cta_minimizers' fast-path flag (same value)
        reports = out.stderr.split("WARNING: ThreadSanitizer: data race")[1:]
        unexpected = [r for r in reports if not re.search(r"#0 (cluster_kernel|cta_minimizers)\(", r)]
        assert not unexpected, unexpected[0][:3000]
    got = {m.group(1): [int(x) for x in m.groups()[1:]] for m in re.finditer(r"(\w+): pairs=(\d+) records=(\d+) tier0=(\d+) tier1=(\d+) tier2=(\d+)", out.stdout)}
    assert got["real_tiers"][1] > 45 and got["real_tiers"][3] > 5, out.stdout                      # records; pairs that climbed to the second tier
    assert got["small_first_tier"][1] > 30 and got["small_first_tier"][3] > 20 and got["small_first_tier"][4] > 3, out.stdout   # CTA kernels, up to the last tier
    assert got["atac_trimming"][1] > 20 and got["hic_split"][1] > 18 and got["single_end"][1] > 25, out.stdout
    assert got["hic_split_cta"][3] > 3 and got["single_end_cta"][3] > 6 and got["sam_cores"][1] > 25 and got["sam_cores_single_end"][1] > 20 and got["heavy_repeats"][4] > 3 and got["front_end_only"][1] > 5000 and got["front_end_k21_w10"][1] > 800 and got["front_end_k16_w5"][1] > 1500, out.stdout
