// chromap_b200 — overflow tiers: draft mappings (draft_mapping_generator.cc:9-357) and best-pair statistics
// (mapping_generator.h:160-197, 346-484) for one read / one pair by one CTA, every order-dependent rule of the
// reference restated so that all threads work.  File:line citations are into the reference's src/.
#pragma once
#include "cta_pair_candidates.cuh"

// Tally (min, #min, second distinct min, #second) of a multiset; the reference builds it one value at a time
// (draft_mapping_generator.cc:213-230), the result does not depend on the order, so partial tallies can be merged.
__device__ __forceinline__ Tally tally_merge(const Tally &a, const Tally &b, int sentinel) {
  Tally r;
  r.min_err = min(a.min_err, b.min_err);
  r.n_best = (a.min_err == r.min_err ? a.n_best : 0) + (b.min_err == r.min_err ? b.n_best : 0);
  // candidates for the second distinct value: whatever of {a.min, a.second, b.min, b.second} is above the minimum
  int s = sentinel;
  if (a.min_err > r.min_err && a.n_best > 0) s = min(s, a.min_err);
  if (b.min_err > r.min_err && b.n_best > 0) s = min(s, b.min_err);
  if (a.n_second_best > 0) s = min(s, a.second_min_err);
  if (b.n_second_best > 0) s = min(s, b.second_min_err);
  r.second_min_err = s;
  int n = 0;
  if (a.min_err == s && a.min_err > r.min_err) n += a.n_best;
  if (b.min_err == s && b.min_err > r.min_err) n += b.n_best;
  if (a.second_min_err == s) n += a.n_second_best;
  if (b.second_min_err == s) n += b.n_second_best;
  r.n_second_best = n;
  return r;
}
__device__ __forceinline__ Tally cta_tally_reduce(Tally t, int sentinel, Tally *s_t /* one per warp */) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Tally u;
    u.min_err = __shfl_down_sync(0xffffffffu, t.min_err, o); u.second_min_err = __shfl_down_sync(0xffffffffu, t.second_min_err, o);
    u.n_best = __shfl_down_sync(0xffffffffu, t.n_best, o); u.n_second_best = __shfl_down_sync(0xffffffffu, t.n_second_best, o);
    t = tally_merge(t, u, sentinel);
  }
  if ((threadIdx.x & 31) == 0) s_t[threadIdx.x >> 5] = t;
  __syncthreads();
  Tally r = s_t[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = tally_merge(r, s_t[i], sentinel);
  __syncthreads();
  return r;
}

// GenerateDraftMappings for one read (non-split).  Candidates are sorted cooperatively (count descending, position
// ascending, candidate.h:23-33).  The reference then verifies the VALID candidates (draft_mapping_generator.cc:59-70) in
// groups of `lanes`; after a full group any failing member sets threshold = its count, and the scan over the sorted
// list stops at the first candidate — valid or not — whose count is below the threshold (:186-188, :254-256); a trailing
// partial group is verified without the rule (:308-356); with fewer than `lanes` candidates there is no rule at all.
// Because counts only decrease along the list, the threshold can only ever be set to ONE value T: the count of the last
// failing member of the first full group that contains a failure; later failures carry the same count.  So
//   taken = valid candidates up to the end of that group, then valid candidates at indices < stop,
//   stop  = first index behind the group whose count is < T.
// The CTA walks the compacted list of valid candidates NT at a time (NT is a multiple of `lanes`, so groups never
// straddle a step), one banded alignment per thread; the step that finds the failing group fixes `stop`, and the walk
// ends at the first step that starts at or beyond it.  Accepted mappings are written in list order (prefix sum per
// step), the error tally is merged at the end.  Work the reference would have skipped is limited to one step.
#define VERIFY_NT_MAX 256  // threads of verify_cta_kernel at most
__global__ void __launch_bounds__(VERIFY_NT_MAX) verify_cta_kernel(DevParams P, DevRef R, DevBatch B, Scratch S, Counters *ctr, int sm_cap) {
  extern __shared__ u64 smk[];  // [sm_cap] sort keys, afterwards the list of valid candidate indices (u16) | [sm_cap] sort tags | read codes
  u8 *smt = (u8 *)(smk + sm_cap);
  u8 *s_fwd = smt + sm_cap, *s_neg = s_fwd + S.caps.maxmm;  // base codes of the read and of its reverse complement
  __shared__ int s_i[8];
  __shared__ int s_warp[VERIFY_NT_MAX / 32];
  __shared__ Tally s_t[VERIFY_NT_MAX / 32];
  const int NT = blockDim.x;  // 128 in the middle tier, 256 in the last one (a multiple of the group size either way)
  const int sr = blockIdx.x, tid = threadIdx.x;
  const int slot = sr >> 1, mate = sr & 1;
  if (tid == 0) s_i[0] = S.pmeta[slot].status;  // the mate's CTA may flag the pair concurrently
  __syncthreads();
  if (s_i[0] != ST_OK || (P.se && mate == 1)) return;
  const int pair = slot_pair(S, slot);
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  const u8 *read = read_ptr(B, pair, mate);
  const int L = rm.len, e = P.e;
  u64 *mp[2] = {S.map_pos + map_base(0, c, sr, 0), S.map_pos + map_base(0, c, sr, 1)};
  short *me[2] = {S.map_err + map_base(0, c, sr, 0), S.map_err + map_base(0, c, sr, 1)};
  u64 *cp[2] = {S.cand_pos + cand_base(0, c, sr, 0, 0), S.cand_pos + cand_base(0, c, sr, 0, 1)};
  u8 *cc[2] = {S.cand_cnt + cand_base(0, c, sr, 0, 0), S.cand_cnt + cand_base(0, c, sr, 0, 1)};
  const int nc[2] = {rm.n_cand[0], rm.n_cand[1]};
  if (nc[0] + nc[1] == 1) {  // fast path (draft_mapping_generator.cc:72-157): the only candidate carries every minimizer
    const int strand = nc[0] == 1 ? 0 : 1;
    if (cc[strand][0] == rm.n_mm) {
      const u64 cpos = cp[strand][0];
      const u32 rid = (u32)(cpos >> 32);
      const u32 pos = strand == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
      const bool ok = valid_cand(e, R.len[rid], pos, (u32)L);
      __syncthreads();
      if (tid == 0) {
        rm.min_err = 0; rm.n_best = 1; rm.second_min_err = e + 1; rm.n_second_best = 0;
        if (ok) {
          mp[strand][0] = strand == 0 ? cpos + (u64)L - 1 : cpos;
          me[strand][0] = 0;
          rm.n_map[strand] = 1; rm.n_map[1 - strand] = 0;
        }
      }
      if (ok) return;
    }
  }
  for (int i = tid; i < L; i += NT) {
    const u32 b = base_code(read[i]);
    s_fwd[i] = (u8)b;
    s_neg[L - 1 - i] = (u8)(b < 4 ? 3u ^ b : 4u);
  }
  auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };
  cta_sort_pairs<u8>(cp[0], cc[0], nc[0], ~0ull, (u8)0, cless, smk, smt, sm_cap);
  cta_sort_pairs<u8>(cp[1], cc[1], nc[1], ~0ull, (u8)0, cless, smk, smt, sm_cap);
  unsigned short *vlist = (unsigned short *)smk;  // 4 * sm_cap entries >= cc
  Tally t = {e + 1, e + 1, 0, 0};
  // the fast path may have tallied a zero-error candidate that turned out invalid: the reference keeps that tally
  // (draft_mapping_generator.cc:100-104 updates min_num_errors before the validity test) and goes on to the full scan
  if (tid == 0 && nc[0] + nc[1] == 1 && cc[nc[0] == 1 ? 0 : 1][0] == rm.n_mm) { t.min_err = 0; t.n_best = 1; }
  u32 n_ver = 0;
  int nm[2] = {0, 0};
  for (int s = 0; s < 2; ++s) {
    const int n = nc[s];
    if (n == 0) continue;
    // compacted list of valid candidates, in list order
    const int C = (n + NT - 1) / NT;
    const int r0 = min(n, tid * C), r1 = min(n, r0 + C);
    int mine = 0;
    for (int i = r0; i < r1; ++i) {
      const u64 cpos = cp[s][i];
      const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
      mine += valid_cand(e, R.len[(u32)(cpos >> 32)], pos, (u32)L) ? 1 : 0;
    }
    int nv;
    int at = cta_scan_add(mine, s_warp, &nv);
    for (int i = r0; i < r1; ++i) {
      const u64 cpos = cp[s][i];
      const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
      if (valid_cand(e, R.len[(u32)(cpos >> 32)], pos, (u32)L)) vlist[at++] = (unsigned short)i;
    }
    __syncthreads();
    const bool ruled = n >= P.lanes;            // the group / threshold rule applies
    const int n_full = nv / P.lanes * P.lanes;  // members of full groups
    int stop = n;                               // candidates at list indices >= stop are not taken ...
    int free_until = 0;                         // ... except those of rank < free_until (the failing group itself)
    int out_base = 0;
    for (int v0 = 0; v0 < nv; v0 += NT) {
      if ((int)vlist[v0] >= stop && v0 >= free_until) break;
      const int v = v0 + tid;
      int err = e + 1, endp = 0, idx = 0;
      u64 cpos = 0;
      if (v + NT < nv) {  // the window this thread aligns in the next step: request its lines now (a cold window is a DRAM round trip)
        const u64 nx = cp[s][vlist[v + NT]];
        const u32 npos = s == 0 ? (u32)nx : (u32)nx - (u32)L + 1u;
        prefetch_span(R.seq + R.off[(u32)(nx >> 32)] + npos - e, L + 2 * e);
      }
      if (v < nv) {
        idx = vlist[v];
        if (idx < stop || v < free_until) {
          cpos = cp[s][idx];
          const u32 rid = (u32)(cpos >> 32);
          const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
          const u8 *win = R.seq + R.off[rid] + pos - e;
          prefetch_span(win, L + 2 * e);
          const u8 *txt = s == 0 ? s_fwd : s_neg;
          err = banded_align(e, L, [&](int q) { return base_code(__ldg(win + q)); }, [&](int q) { return (u32)txt[q]; }, &endp);
          ++n_ver;
        } else idx = -1;
      } else idx = -1;
      if (ruled && stop == n && free_until == 0) {
        // first full group with a failure in this step, the last failing member's count, and where the scan stops
        const bool failing = idx >= 0 && v < n_full && err > e;
        const unsigned fm = __ballot_sync(0xffffffffu, failing);
        if ((tid & 31) == 0) s_warp[tid >> 5] = (int)fm;
        __syncthreads();
        int first_fail = -1;
#pragma unroll
        for (int w = 0; w < (NT >> 5); ++w) if (first_fail < 0 && s_warp[w]) first_fail = v0 + w * 32 + __ffs((unsigned)s_warp[w]) - 1;
        if (first_fail >= 0) {
          const int g0 = first_fail / P.lanes * P.lanes, g1 = g0 + P.lanes;  // ranks of the failing group (inside this step)
          int last_fail = first_fail;
          for (int q = g0; q < g1; ++q) { const int w = (q - v0) >> 5, b = (q - v0) & 31; if ((s_warp[w] >> b) & 1) last_fail = q; }
          const int T = cc[s][vlist[last_fail]];
          int lo = (int)vlist[g1 - 1] + 1, hi = n;  // first index behind the group with count < T (counts descend)
          while (lo < hi) { const int m = (lo + hi) >> 1; if ((int)cc[s][m] < T) hi = m; else lo = m + 1; }
          stop = lo;
          free_until = g1;
        }
        __syncthreads();
      }
      const bool taken = idx >= 0 && (idx < stop || v < free_until);
      const bool pass = taken && err <= e;
      int tot;
      const int o = out_base + cta_scan_add(pass ? 1 : 0, s_warp, &tot);
      if (pass) {
        tally(t, err);
        if (o < c.mc) {
          mp[s][o] = s == 0 ? cpos - (u64)e + (u64)endp : cpos - (u64)L + 1 - (u64)e + (u64)endp;
          me[s][o] = (short)err;
        }
      }
      out_base += tot;
    }
    nm[s] = out_base;
    __syncthreads();
  }
  const Tally tt = cta_tally_reduce(t, e + 1, s_t);
  if (n_ver) agg_add(&ctr->n_verified, (u64)n_ver);
  if (tid != 0) return;
  if (nm[0] > c.mc || nm[1] > c.mc) { S.pmeta[slot].status = ST_OVERFLOW; return; }
  rm.n_map[0] = nm[0]; rm.n_map[1] = nm[1];
  rm.min_err = tt.min_err; rm.second_min_err = tt.second_min_err; rm.n_best = tt.n_best; rm.n_second_best = tt.n_second_best;
}

// Best-pair statistics for one pair by one CTA (mapping_generator.h:346-484, non-split).  The reference's two-pointer
// sweep visits, for every mapping i1 of mate 1 in position order, the contiguous run of mate-2 mappings whose end
// positions fall into i1's window: [first j that is not "too far left", first j beyond the window).  Both bounds are
// monotone in i1, so each is a binary search and the (i1, j) pairs can be tallied by all threads independently.
// in_lo(j): mate-2 mapping j lies before i1's window; in_hi(j): j lies inside or before the window's end.
struct SweepWindow {
  u64 ins, ovl;
  u32 L1, L2;
  int s1;
  __device__ __forceinline__ bool before(u64 p1, u64 p2) const { return (s1 == 1 && p1 > p2 + ins - L2) || (s1 == 0 && p1 > p2 + L1 - ovl); }
  __device__ __forceinline__ bool within(u64 p1, u64 p2) const { return (s1 == 0 && p2 <= p1 + ins - L1) || (s1 == 1 && p2 <= p1 + L2 - ovl); }
  __device__ __forceinline__ void range(u64 p1, const u64 *p2, int n2, int *lo, int *hi) const {
    int a = 0, b = n2;
    while (a < b) { const int m = (a + b) >> 1; if (before(p1, p2[m])) a = m + 1; else b = m; }
    *lo = a;
    b = n2;
    while (a < b) { const int m = (a + b) >> 1; if (within(p1, p2[m])) a = m + 1; else b = m; }
    *hi = a;
  }
};

__global__ void __launch_bounds__(CTA_NT) pairing_cta_kernel(DevParams P, Scratch S, int *pair_nbest, int sm_cap) {
  extern __shared__ u64 smk[];
  short *smt = (short *)(smk + sm_cap);
  __shared__ Tally s_t[CTA_NT / 32];
  const int slot = blockIdx.x, tid = threadIdx.x;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status != ST_OK) { if (tid == 0 && pm.status == ST_DROP) pair_nbest[pair] = 0; return; }
  const Caps c = S.caps;
  ReadMeta *rm = S.rmeta + 2 * slot;
  if (P.se) {
    __syncthreads();
    if (tid == 0) {
      if (rm[0].n_map[0] + rm[0].n_map[1] == 0) { pm.status = ST_DROP; pair_nbest[pair] = 0; }
      else {
        pm.min_sum = rm[0].min_err; pm.second_min_sum = rm[0].second_min_err; pm.n_best = rm[0].n_best; pm.n_second_best = rm[0].n_second_best;
        pair_nbest[pair] = rm[0].n_best;
      }
    }
    return;
  }
  if (rm[0].n_map[0] + rm[0].n_map[1] == 0 || rm[1].n_map[0] + rm[1].n_map[1] == 0) {
    __syncthreads();
    if (tid == 0) { pm.status = ST_DROP; pair_nbest[pair] = 0; }
    return;
  }
  auto mless = [](u64 pa, short ea, u64 pb, short eb) { return pa != pb ? pa < pb : ea < eb; };
  u64 *mp[2][2];
  short *me[2][2];
  for (int m = 0; m < 2; ++m)
    for (int s = 0; s < 2; ++s) {
      mp[m][s] = S.map_pos + map_base(0, c, 2 * slot + m, s);
      me[m][s] = S.map_err + map_base(0, c, 2 * slot + m, s);
      cta_sort_pairs<short>(mp[m][s], me[m][s], rm[m].n_map[s], ~0ull, (short)32767, mless, smk, smt, sm_cap);
    }
  const int sentinel = 2 * P.e + 1;
  Tally t = {sentinel, sentinel, 0, 0};
  SweepWindow W;
  W.ins = (u64)P.max_insert; W.ovl = (u64)(u32)P.min_read_len; W.L1 = (u32)rm[0].len; W.L2 = (u32)rm[1].len;
  for (int dir = 0; dir < 2; ++dir) {
    W.s1 = dir;
    const u64 *p1 = mp[0][dir], *p2 = mp[1][1 - dir];
    const short *e1 = me[0][dir], *e2 = me[1][1 - dir];
    const int n1 = rm[0].n_map[dir], n2 = rm[1].n_map[1 - dir];
    for (int i1 = tid; i1 < n1; i1 += CTA_NT) {
      int lo, hi;
      W.range(p1[i1], p2, n2, &lo, &hi);
      const int ea = e1[i1];
      for (int j = lo; j < hi; ++j) tally(t, ea + (int)e2[j]);
    }
  }
  const Tally tt = cta_tally_reduce(t, sentinel, s_t);
  if (tid != 0) return;
  pm.min_sum = tt.min_err; pm.second_min_sum = tt.second_min_err; pm.n_best = tt.n_best; pm.n_second_best = tt.n_second_best;
  pair_nbest[pair] = (tt.n_best > P.drop_rep) ? 0 : tt.n_best;
}

// Record emit for one pair of the overflow tiers by one CTA (mapping_generator.h:486-654).  The reference walks the
// sweep again and reports the best pairs (sum of errors == the minimum) whose running index is in the selection.  Here
// every thread counts the best pairs of its share of mate-1 mappings (windows by binary search as in pairing_cta_kernel),
// a prefix sum gives each share its first running index, and the threads whose share contains a selected index note the
// mappings; threads 0 .. reported-1 then compute one record each.
__global__ void __launch_bounds__(CTA_NT) emit_cta_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutRecord *out,
                                                          int *out_n, Counters *ctr) {
  __shared__ int s_warp[CTA_NT / 32];
  __shared__ int s_i1[CMX_MAX_BEST], s_j[CMX_MAX_BEST], s_sel[CMX_MAX_BEST];
  const int slot = blockIdx.x, tid = threadIdx.x;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status == ST_OVERFLOW) return;
  if (pm.status != ST_OK || pm.n_best > P.drop_rep || pm.n_best == 0) { if (tid == 0) out_n[pair] = 0; return; }
  const Caps c = S.caps;
  const ReadMeta *rm = S.rmeta + 2 * slot;
  const int mb = P.max_best;
  const int to_report = mb < pm.n_best ? mb : pm.n_best;
  if (tid < to_report) s_sel[tid] = pair_sel[(size_t)pair * mb + tid];
  __syncthreads();
  const int min_sum = pm.min_sum;
  SweepWindow W;
  W.ins = (u64)P.max_insert; W.ovl = (u64)(u32)P.min_read_len; W.L1 = (u32)rm[0].len; W.L2 = (u32)rm[1].len;
  int base = 0;  // running index of the first best pair of this direction
  for (int dir = 0; dir < 2; ++dir) {
    if (base > s_sel[to_report - 1]) break;  // every selected index lies in the directions already walked
    W.s1 = dir;
    const u64 *p1 = S.map_pos + map_base(0, c, 2 * slot, dir), *p2 = S.map_pos + map_base(0, c, 2 * slot + 1, 1 - dir);
    const short *e1 = S.map_err + map_base(0, c, 2 * slot, dir), *e2 = S.map_err + map_base(0, c, 2 * slot + 1, 1 - dir);
    const int n1 = rm[0].n_map[dir], n2 = rm[1].n_map[1 - dir];
    const int C = (n1 + CTA_NT - 1) / CTA_NT;
    const int r0 = min(n1, tid * C), r1 = min(n1, r0 + C);
    int mine = 0;
    for (int i1 = r0; i1 < r1; ++i1) {
      int lo, hi;
      W.range(p1[i1], p2, n2, &lo, &hi);
      const int want = min_sum - (int)e1[i1];
      for (int j = lo; j < hi; ++j) mine += (int)e2[j] == want;
    }
    int total;
    int idx = base + cta_scan_add(mine, s_warp, &total);
    if (mine > 0) {
      int r = 0;
      while (r < to_report && s_sel[r] < idx) ++r;
      if (r < to_report && s_sel[r] < idx + mine) {  // a selected index falls into this share: walk it again
        for (int i1 = r0; i1 < r1 && r < to_report; ++i1) {
          int lo, hi;
          W.range(p1[i1], p2, n2, &lo, &hi);
          const int want = min_sum - (int)e1[i1];
          for (int j = lo; j < hi && r < to_report; ++j) {
            if ((int)e2[j] != want) continue;
            if (idx == s_sel[r]) { s_i1[r] = i1 | (dir << 30); s_j[r] = j; ++r; }
            ++idx;
          }
        }
      }
    }
    base += total;
  }
  __syncthreads();
  // best pairs exist for every selected index (the selection never exceeds n_best), so all to_report records are reported
  if (tid < to_report) {
    const int s1 = s_i1[tid] >> 30, i1 = s_i1[tid] & 0x3FFFFFFF, j = s_j[tid];
    const size_t b1 = map_base(0, c, 2 * slot, s1) + i1, b2 = map_base(0, c, 2 * slot + 1, 1 - s1) + j;
    out[(size_t)pair * mb + tid] = pe_record(P, R, B, T, pm, rm, pair, s1, S.map_pos[b1], S.map_err[b1], S.map_pos[b2], S.map_err[b2]);
  }
  if (tid != 0) return;
  out_n[pair] = to_report;
  pm.n_rec = to_report;
  atomicAdd(&ctr->n_mapped, 1ull);
  if (pm.n_best == 1) atomicAdd(&ctr->n_unique, 1ull);
}
