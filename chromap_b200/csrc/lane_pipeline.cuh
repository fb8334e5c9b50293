// chromap_b200 — the launch sequence of one lane's mapping pipeline, host code only: which kernels run in which order, with
// which grids, blocks and shared-memory sizes, and the host decisions between them.  The library (api.cu, run_lane) runs it
// on CUDA streams; the host test of the whole pipeline runs the same sequence on emulated CTAs.  Each supplies an object `x`
// for what differs between the two:
//   x(kernel, grid, block, smem, args...)   launch
//   x.mark(m)                               timing mark m (LaneMark)
//   x.wait_piece(q)                         reads of piece q have landed
//   x.tier(t, n, pair_list)                 tier t's scratch for n pair slots (slot -> pair: pair_list, nullptr = identity)
//   x.list(l, bytes)                        list buffer l (LaneList) of at least `bytes` bytes
//   x.clear_counts(i, n)                    clear the list counters i .. i + n - 1 (LaneArgs::count)
//   x.overflow_count(t)                     pairs that overflowed tier t (counter 0), read back when tier t has run
//   x.sort_list(list, n)                    the overflow list, sorted, as the next tier's pair list
//   x.chunk_starts(chunks)                  the taskloop chunk starts where select_kernel reads them
//   x.emit_on(t), x.emit_join(tiers_used)   the stream of tier t's emission; the join after emission
#pragma once
#include <algorithm>
#include <vector>

#include "pipeline_kernels.cuh"
#include "seed_front.cuh"
#include "cta_pair_candidates.cuh"
#include "cta_verify_pairing.cuh"
#include "sam_kernels.cuh"

#define N_TIERS 3

enum LaneMark { MARK_TIER, MARK_FRONT, MARK_SEED, MARK_PC, MARK_VER, MARK_PAIR, MARK_SELECT, MARK_EMIT };
enum LaneList { LIST_RESCUE, LIST_VERIFY, LIST_EMIT, LIST_OVERFLOW };  // LIST_OVERFLOW + t: the pairs that overflowed tier t

// The kernels' parameters from the library's cmx_params or the oracle's orc_params (the field names agree).
template <typename Params>
inline DevParams dev_params(const Params &p, int k, int w) {
  DevParams d;
  d.e = p.error_threshold; d.min_seeds = p.min_num_seeds; d.f0 = p.max_seed_freq0; d.f1 = p.max_seed_freq1;
  d.max_best = p.max_num_best_mappings; d.max_insert = p.max_insert_size; d.min_read_len = p.min_read_length;
  d.drop_rep = p.drop_repetitive_reads; d.trim = p.trim_adapters; d.k = k; d.w = w;
  d.lanes = p.error_threshold < 8 ? 8 : 4;  // mapping_parameters.h:80-88
  d.split = p.split_alignment;
  d.se = p.single_end;
  return d;
}

// Tier 0's hit capacity: 64, and above 160 bases as many hits per base as at 160 (a read has about 2L / (w + 1) minimizers,
// each with one hit or more), in whole cluster-kernel rows of 16, at most TIER0_HC_MAX: cluster_kernel holds a read's hits
// in shared memory, hc x CLUSTER_NT x 8 bytes per CTA (192 KB at the cap).
#define TIER0_HC_MAX 192
inline int tier0_hits(int max_read_length) { return std::min(TIER0_HC_MAX, std::max(64, (max_read_length * 2 / 5 + 15) / 16 * 16)); }

// Scratch capacities of tier t for reads of up to max_read_length bases: {minimizers, hits, candidates, draft mappings}.
inline Caps tier_caps(int max_read_length, int t) {
  const int mrl = max_read_length;
  const Caps c[N_TIERS] = {{mrl, tier0_hits(mrl), 32, 32}, {mrl * 2, 1024, 256, 256}, {mrl * 4, 65536, 8192, 8192}};
  return c[t];
}

// Task chunks of `#pragma omp taskloop grainsize(5000)` (chromap.h:892) over one reference batch of n pairs
// as cut by libgomp: num_tasks = n/5000 (min 1), chunk = n/num_tasks, first n%num_tasks chunks one longer.
inline void taskloop_chunks(u32 base, u32 n, std::vector<int> &starts) {
  u32 nt = n / 5000;
  if (nt < 1) nt = 1;
  const u32 chunk = n / nt, rem = n % nt;
  u32 s = base;
  for (u32 t = 0; t < nt; ++t) { starts.push_back((int)s); s += chunk + (t < rem ? 1 : 0); }
}

// What a lane maps and where the per-pair results go (device pointers).
struct LaneArgs {
  DevParams P;
  DevIndex ix;
  DevRef R;
  DevBatch B;  // the lane's pairs
  MapqTables T;
  const u32 *mt_init;
  Counters *ctr;
  int *count;  // [4] list counters: 0 overflow, 1 rescue, 2 verify / emit's tracebacks, 3 cluster's second pass
  int *nbest, *sel, *out_n;
  void *out_rec;  // OutRecord, OutPairs (split alignment) or OutSam (sam)
  bool sam;
  int max_read_length;
};

struct LaneTiers {
  Scratch S[N_TIERS];
  int used = 0;
  int n_left = 0;  // pairs that overflowed the last tier
};

static const int LANE_TB = 128;

// The barcode gate of n barcodes: keys, accept flags and the two counters.  At --bc-error-threshold 2 the barcodes that need a
// search are corrected by barcode_correct2_kernel: first with hit lists in shared memory, then the few with more hits than
// those hold, with a slab per warp.  ctr's list counters start at zero.
template <class X>
void lane_barcodes(X &x, const DevWhitelist &W, const u8 *bc_seq, const u8 *bc_qual, int bc_len, int n, u64 *bc_key, u8 *bc_ok, Counters *ctr) {
  x(barcode_kernel, (n + 127) / 128, 128, 0, W, bc_seq, bc_qual, bc_len, n, bc_key, bc_ok, ctr);
  if (!W.active || W.err_threshold != 2) return;
  x(barcode_correct2_kernel, std::min((n + BC2_WARPS - 1) / BC2_WARPS, BC2_GRID_MAX), BC2_WARPS * 32, 0, W, bc_seq, bc_qual, bc_len, bc_key, bc_ok, ctr, 0);
  x(barcode_correct2_kernel, BC2_SLAB_WARPS / BC2_WARPS, BC2_WARPS * 32, 0, W, bc_seq, bc_qual, bc_len, bc_key, bc_ok, ctr, 1);
}

// Tier 0 for all pairs, and its front end: [adapter trimming] + length filter + minimizers + index probe in one kernel over
// staged read tiles (seed_front.cuh).  When the reads arrive in pieces of `piece` pairs, one grid per piece starts as soon
// as the piece has landed; the rest of the upload hides behind it.  grid_cap: seed_front_kernel's persistent grid.
template <class X>
Scratch lane_front(X &x, const LaneArgs &a, u32 piece, int grid_cap) {
  const DevParams &P = a.P;
  const u32 n = a.B.n_pairs;
  const Scratch S = x.tier(0, (int)n, nullptr);
  x.mark(MARK_TIER);
  const size_t sf_smem = seed_front_smem_bytes(S.caps.maxmm);
  for (u32 q = 0, p0 = 0; p0 < n; ++q, p0 += piece) {
    const u32 np = std::min(piece, n - p0);
    x.wait_piece(q);
    if (P.trim) {
      Scratch V = S;
      V.n_slots = (int)np; V.rmeta += 2 * (size_t)p0; V.pmeta += p0;
      DevBatch Bq = a.B;
      if (Bq.bc_ok) Bq.bc_ok += p0;
      Bq.off1 += p0; Bq.off2 += p0; Bq.n_pairs = np;
      x(prep_kernel, (int)((np + LANE_TB - 1) / LANE_TB), LANE_TB, 0, P, Bq, V);
    }
    // packed-key scan for k = 17, w = 7 and reads the key layout can address (minimizers.cuh); the run-time scan otherwise
    const auto front = P.k == 17 && P.w == 7 && S.caps.maxmm < (1 << 18) ? seed_front_kernel<true> : seed_front_kernel<false>;
    x(front, std::min((int)((np + SF_TILE - 1) / SF_TILE), grid_cap), SF_NT, sf_smem, P, a.ix, a.B, S, a.ctr, P.trim ? 1 : 0, (int)p0, (int)(p0 + np));
  }
  return S;
}

// Tier 0 from the front end's records on (S: as lane_front left it), then the overflow tiers, one CTA per read / pair with
// shared-memory sort buffers sized to the tier, each on the pairs the tier before could not hold.
template <class X>
LaneTiers lane_tiers(X &x, const LaneArgs &a, Scratch S) {
  const DevParams &P = a.P;
  const int TB = LANE_TB;
  int *cnt = a.count;
  LaneTiers r;
  for (int t = 0;; ++t) {
    const int n = S.n_slots;
    r.S[t] = S;
    if (t == 0) {
      int *rescue = (int *)x.list(LIST_RESCUE, (size_t)n * 4), *verify = (int *)x.list(LIST_VERIFY, (size_t)n * 8);  // verify: cluster's, then verify's
      x.clear_counts(1, 3);
      x.mark(MARK_FRONT);
      // first-pass tile: enough rows for a typical read (about 2L/(w+1) minimizers, most of them single hits)
      int rows0 = (2 * a.max_read_length / (P.w + 1) + 15) / 16 * 16;  // 16 rows at 2x50, 48 at 2x150
      rows0 = std::max(16, std::min(rows0, S.caps.hc));
      const int cg = (2 * n + CLUSTER_NT - 1) / CLUSTER_NT;
      x(cluster_kernel, cg, CLUSTER_NT, (size_t)rows0 * CLUSTER_NT * 8, P, a.ix, S, a.ctr, 0, rows0, verify, cnt + 3);
      if (rows0 < S.caps.hc) x(cluster_kernel, cg, CLUSTER_NT, (size_t)S.caps.hc * CLUSTER_NT * 8, P, a.ix, S, a.ctr, 1, S.caps.hc, verify, cnt + 3);
      x.mark(MARK_SEED);
      x(pair_candidates_kernel, (n + TB - 1) / TB, TB, 0, P, a.ix, S, a.ctr, 0, rescue, cnt + 1);
      x(pair_candidates_kernel, (n + 63) / 64, 64, 0, P, a.ix, S, a.ctr, 1, rescue, cnt + 1);
      x.mark(MARK_PC);
      if (P.split) x(verify_split_kernel, (2 * n + TB - 1) / TB, TB, 0, P, a.R, a.B, S, a.ctr);
      else {
        x(verify_kernel, (2 * n + TB - 1) / TB, TB, 0, P, a.R, a.B, S, a.ctr, 0, verify, cnt + 2);
        x(verify_kernel, (2 * n + 63) / 64, 64, (size_t)2 * S.caps.maxmm * 64, P, a.R, a.B, S, a.ctr, 1, verify, cnt + 2);
      }
      x.mark(MARK_VER);
      if (P.split) x(pairing_split_kernel, (n + TB - 1) / TB, TB, 0, P, S, a.nbest);
      else x(pairing_kernel, (n + TB - 1) / TB, TB, 0, P, S, a.nbest);
      x.mark(MARK_PAIR);
    } else {
      auto cap_of = [](int c_) { int c = 1; while (c < c_) c <<= 1; return std::min(c, CTA_SORT_SMEM_MAX); };
      const Caps &c = S.caps;
      const int c_seed = cap_of(2 * c.hc), c_pc = cap_of(c.hc), c_ver = cap_of(c.cc), c_pair = cap_of(c.mc);
      x(prep_kernel, (n + TB - 1) / TB, TB, 0, P, a.B, S);
      x(seed_cta_kernel, 2 * n, CTA_NT, (size_t)c_seed * 11 + (size_t)(c.maxmm + 1) * 12 + 16, P, a.ix, a.B, S, r.S[0], a.ctr, c_seed);
      x.mark(MARK_SEED);
      // the last tier's shared-memory lists leave room for two CTAs per SM only: sixteen warps each instead of four keep as
      // many dependent occurrence-list searches in flight as the smaller tiers do
      const int lcap = std::min(c.cc, 512), fcap = 2 * c.cc;
      const size_t pc_smem = pair_candidates_cta_smem(c_pc, lcap, c.maxmm, fcap);
      x(pair_candidates_cta_kernel, n, pc_smem > 64 * 1024 ? PC_CTA_NT_MAX : CTA_NT, pc_smem, P, a.ix, S, a.ctr, c_pc, lcap, fcap, (const int *)nullptr, (const int *)nullptr);
      x.mark(MARK_PC);
      if (P.split) x(verify_split_cta_kernel, 2 * n, CTA_NT, (size_t)c_ver * 9, P, a.R, a.B, S, a.ctr, c_ver);
      else x(verify_cta_kernel, 2 * n, c.cc > 1024 ? VERIFY_NT_MAX : CTA_NT, (size_t)c_ver * 9 + 2 * (size_t)c.maxmm + 16, P, a.R, a.B, S, a.ctr, c_ver);
      x.mark(MARK_VER);
      if (P.split) x(pairing_split_kernel, (n + TB - 1) / TB, TB, 0, P, S, a.nbest);
      else x(pairing_cta_kernel, n, CTA_NT, (size_t)c_pair * 10, P, S, a.nbest, c_pair);
      x.mark(MARK_PAIR);
    }
    int *ovf = (int *)x.list(LIST_OVERFLOW + t, (size_t)n * 4);
    x.clear_counts(0, 1);
    x(collect_overflow_kernel, (n + 255) / 256, 256, 0, S, ovf, cnt);
    const int n_ovf = x.overflow_count(t);
    r.used = t + 1;
    if (n_ovf == 0 || t + 1 == N_TIERS) { r.n_left = n_ovf; return r; }
    // deterministic order for the next tier: the list sorted (atomic append order is arbitrary)
    S = x.tier(t + 1, n_ovf, x.sort_list(ovf, n_ovf));
    x.mark(MARK_TIER);
  }
}

// Multi-mapper sampling, one warp per taskloop chunk of every reference batch (batch_size pairs) of the lane; then the
// emission of every tier used, the overflow tiers' (few pairs, long per-thread sweeps) beside tier 0's.
template <class X>
void lane_emit(X &x, const LaneArgs &a, const LaneTiers &tiers, u32 batch_size) {
  const DevParams &P = a.P;
  const int TB = LANE_TB;
  const u32 n = a.B.n_pairs;
  std::vector<int> chunks;
  for (u32 b0 = 0; b0 < n; b0 += batch_size) taskloop_chunks(b0, std::min(batch_size, n - b0), chunks);
  const int n_chunks = (int)chunks.size();
  chunks.push_back((int)n);
  x.mark(MARK_SELECT);
  x(select_kernel, (n_chunks + 3) / 4, 128, 0, P, n_chunks, x.chunk_starts(chunks), (const int *)a.nbest, a.sel, a.mt_init);
  x.mark(MARK_EMIT);
  for (int t = tiers.used - 1; t >= 0; --t) {
    const Scratch &S = tiers.S[t];
    const int g = (S.n_slots + TB - 1) / TB;
    x.emit_on(t);
    if (P.split) x(emit_split_kernel, g, TB, 0, P, a.R, a.B, a.T, S, a.sel, (OutPairs *)a.out_rec, a.out_n, a.ctr);
    else if (a.sam) {
      // the long instance's direction matrix is twice the local memory of the short one: only contexts sized for it use it
      const bool sam_long = a.max_read_length > SAM_MAX_L;
      const auto emit_sam = P.se ? (sam_long ? emit_sam_se_kernel<SAM_MAX_L_LONG> : emit_sam_se_kernel<SAM_MAX_L>)
                                 : (sam_long ? emit_sam_kernel<SAM_MAX_L_LONG> : emit_sam_kernel<SAM_MAX_L>);
      x(emit_sam, g, TB, 0, P, a.R, a.B, a.T, S, a.sel, (OutSam *)a.out_rec, a.out_n, a.ctr);
    }
    else if (P.se) x(emit_se_kernel, g, TB, 0, P, a.R, a.B, a.T, S, a.sel, (OutRecord *)a.out_rec, a.out_n, a.ctr);
    else if (t > 0) x(emit_cta_kernel, S.n_slots, CTA_NT, 0, P, a.R, a.B, a.T, S, a.sel, (OutRecord *)a.out_rec, a.out_n, a.ctr);
    else {
      int4 *dp = (int4 *)x.list(LIST_EMIT, (size_t)S.n_slots * P.max_best * sizeof(int4));
      int *dp_count = a.count + 2;  // (verify's list counter: free by now)
      x.clear_counts(2, 1);
      x(emit_kernel, g, TB, 0, P, a.R, a.B, a.T, S, a.sel, (OutRecord *)a.out_rec, a.out_n, a.ctr, dp, dp_count);
      // the pairs whose start coordinates need the bit-vector traceback (indels); the grid covers the worst case, idle threads leave at once
      x(emit_dp_kernel, (int)(((size_t)S.n_slots * P.max_best + TB - 1) / TB), TB, 0, P, a.R, a.B, a.T, S, (OutRecord *)a.out_rec, (const int4 *)dp, (const int *)dp_count);
    }
  }
  x.emit_join(tiers.used);
}
