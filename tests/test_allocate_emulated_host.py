"""--allocate-multi-mappings: the kernels of chromap_b200/csrc/allocate.cuh run UNCHANGED on the host emulation (tests/cta_emu.h),
in cmx_allocate_multi_mappings_gpu's order with std::stable_sort in CUB's place, against the restatement of the reference's
AllocateMultiMappings in tests/allocate_oracle.h (an implicit interval tree, std::mt19937, std::discrete_distribution) on random
sorted record sets; and the per-read draw (al_draw) against std::discrete_distribution on a million random weight vectors."""
import os

from tests import emu

HERE = os.path.dirname(os.path.abspath(__file__))

MAIN = r'''
#include "ALLOC_ORACLE_H"
template <typename F> static void launch(size_t n, F body) { emu_grid_serial((int)((n + 255) / 256), 256, body); }
// CUB SortPairs / SortKeys: stable by key
template <typename K> static std::vector<u32> stable_order(const std::vector<K> &keys) {
  std::vector<u32> ord(keys.size());
  std::iota(ord.begin(), ord.end(), 0u);
  std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return keys[a] < keys[b]; });
  return ord;
}
static u32 mk_len(std::mt19937 &g) { return 50 + g() % 400; }
// a sorted, duplicate-free record set: n_seq sequences (the last has no uni record), starts in [base, base + span) so that
// many are equal (half of them moved by hop when it is not 0), reads with 1..max_cand candidates (mapq < 4), uni records (mapq >= 4)
static std::vector<PpRecord> random_set(std::mt19937 &g, int n_uni, int n_reads, int max_cand, int n_seq, u32 base, u32 span, u32 hop) {
  std::vector<PpRecord> r;
  auto rec = [&](u32 read_id, u32 rid, u32 mapq) {
    PpRecord x{};
    x.w[0] = read_id; x.w[1] = rid; x.w[2] = base + g() % span + (hop && (g() & 1) ? hop : 0u);
    x.w[3] = mk_len(g) | (mapq << 16) | ((g() & 1) << 24);
    x.w[4] = (mapq >= 4 ? 1u : (g() % 4 == 0)) | (1u << 8) | ((30 + g() % 20) << 16);
    x.w[5] = 30 + g() % 20;
    r.push_back(x);
  };
  u32 id = 0;
  for (int i = 0; i < n_uni; ++i) rec(id++, g() % (n_seq - 1), 4 + g() % 57);
  for (int i = 0; i < n_reads; ++i, ++id) {
    const int c = 1 + (int)(g() % max_cand);
    for (int k = 0; k < c; ++k) rec(id, g() % n_seq, g() % 4);
  }
  std::sort(r.begin(), r.end(), [](const PpRecord &a, const PpRecord &b) {
    auto key = [](const PpRecord &x) { return std::make_tuple(x.w[1], x.w[2], pe_len(x), pe_mapq(x), pe_dir(x), pe_uniq(x), x.w[0]); };
    return key(a) < key(b);
  });
  return r;
}
static long bad = 0;
static void check(bool ok, const char *what, long a, long b) { if (!ok) { if (bad < 8) printf("MISMATCH %s: %ld vs %ld\n", what, a, b); ++bad; } }

// the device sequence of cmx_allocate_multi_mappings_gpu on sorted records: keep flags and stats
static void device_flow(const std::vector<PpRecord> &rec, u32 d, int seed, std::vector<u8> &keep, orc_alloc_stats &st, std::vector<u32> &weight_out,
                        std::vector<u32> &midx_out) {
  const size_t n = rec.size();
  std::vector<u8> uni(n), multi(n);
  std::vector<u64> ks(n), ke(n);
  launch(n, [&]() { al_split_kernel(rec.data(), n, uni.data(), multi.data(), ks.data(), ke.data()); });
  std::vector<u64> us, ue_s;
  std::vector<u32> midx;
  for (size_t i = 0; i < n; ++i) { if (uni[i]) { us.push_back(ks[i]); ue_s.push_back(ke[i]); } if (multi[i]) midx.push_back((u32)i); }
  std::vector<u64> ue = ue_s;
  { auto o = stable_order(ue_s); for (size_t i = 0; i < o.size(); ++i) ue[i] = ue_s[o[i]]; }
  const u32 n_uni = (u32)us.size(), m = (u32)midx.size();
  std::vector<u32> w(m), rk(m);
  launch(m, [&]() { al_count_kernel(rec.data(), midx.data(), m, us.data(), ue_s.data(), ue.data(), n_uni, d, w.data(), rk.data()); });
  std::vector<u32> perm = stable_order(rk), rk2(m), ws(m);
  for (u32 i = 0; i < m; ++i) rk2[i] = rk[perm[i]];
  std::vector<u8> head(m);
  launch(m, [&]() { al_head_kernel(rk2.data(), perm.data(), w.data(), m, head.data(), ws.data()); });
  std::vector<u32> rs;
  for (u32 i = 0; i < m; ++i) if (head[i]) rs.push_back(i);
  const u32 n_reads = (u32)rs.size();
  std::vector<u32> draws(n_reads), didx(n_reads);
  std::vector<u8> kept(n_reads);
  launch(n_reads, [&]() { al_read_kernel(rs.data(), n_reads, m, ws.data(), draws.data(), kept.data()); });
  u64 n_draws = 0;
  for (u32 r = 0; r < n_reads; ++r) { didx[r] = (u32)n_draws; n_draws += draws[r]; }
  std::vector<u32> stream(2 * n_draws + 1);
  if (n_draws) {
    u32 mt[624];
    mt_seed_fill(mt, (u32)seed);
    emu_launch(256, [&]() { al_mt_kernel(mt, 2 * n_draws, stream.data()); });
  }
  keep = uni;
  launch(n_reads, [&]() { al_draw_kernel(rs.data(), n_reads, m, ws.data(), perm.data(), midx.data(), draws.data(), didx.data(), kept.data(), stream.data(), keep.data()); });
  std::vector<PpRecord> out;
  for (size_t i = 0; i < n; ++i) if (keep[i]) out.push_back(rec[i]);
  unsigned long long n_unique = 0;
  const size_t n2 = out.size();
  out.resize(n2 + 256);
  emu_grid((int)((n2 + 255) / 256), 256, [&]() { al_unique_count_kernel(out.data(), n2, &n_unique); });
  u64 n_kept = 0;
  for (u32 r = 0; r < n_reads; ++r) n_kept += kept[r];
  st = orc_alloc_stats{m, n_kept, n_reads - n_kept, n_draws, n_unique, n2 - n_unique};
  weight_out = w; midx_out = midx;
}

int main() {
  std::mt19937 g(131);
  long cases = 0, draws_total = 0, weights_checked = 0, wrapped_overlaps = 0;
  g_emu_leavable = true;
  // ---- the draw against std::discrete_distribution + std::mt19937, a million weight vectors of 1..16 entries, zeros included
  {
    std::mt19937 gen(11);
    std::vector<u32> w;
    for (int it = 0; it < 1000000; ++it) {
      const int len = 1 + (int)(g() % 16);
      const int mode = (int)(g() % 4);
      w.resize(len);
      for (auto &x : w) x = mode == 0 ? g() % 3 : mode == 1 ? (g() % 2 ? 0u : g() % 1000) : mode == 2 ? g() % 100000 : (g() % 8 ? 1u : 0xFFFFFFu);
      u32 sum = 0;
      for (u32 x : w) sum += x;
      if (sum == 0) continue;  // the reference does not draw
      std::mt19937 copy = gen;
      std::discrete_distribution<uint32_t> dist(w.begin(), w.end());
      const u32 want = dist(gen);
      if (len < 2) { check(want == 0 && copy == gen, "single-candidate draw consumed the generator", want, 0); continue; }
      const u32 g1 = copy(), g2 = copy();
      check(copy == gen, "two outputs per draw", 0, 0);
      check(al_draw(w.data(), (u32)len, g1, g2) == want, "al_draw", al_draw(w.data(), (u32)len, g1, g2), want);
      ++draws_total;
    }
  }
  // ---- the kernels against the restatement
  struct Set { int n_uni, n_reads, max_cand, n_seq; u32 base, span, hop = 0; };
  const Set sets[] = {
      {3000, 1500, 5, 4, 1000, 2000},                   // many equal starts, dense overlaps
      {800, 2000, 8, 5, 0, 200000},                     // sparse: many reads without overlaps, one candidate reads
      {300, 600, 3, 3, 4294967295u - 2000u, 1200},      // at the top of the uint32 range: end + d wraps
      {5000, 16000, 4, 3, 0, 60000},                    // more than 10,000 draws: the stream crosses many 624-word blocks
      {200, 300, 20, 2, 5000, 3000},                    // reads with many candidates
      {0, 800, 4, 3, 0, 5000},                          // no uni record at all: every read is dropped, nothing is kept
      {3000, 1500, 3, 3, 0, 4294966000u},               // starts over the whole uint32 range
      {2000, 1500, 3, 3, 1000, 2000, 2147483648u},      // two clusters 2^31 apart: at d near 2^31 wrapped queries of one reach the other
  };
  // 2^31 - 300: end + d wraps for every multi record up to 600 long, and qs - qe = 600 - length is short enough for a uni
  // record to straddle it (2^31 - 1 leaves such overlaps to lengths <= 2)
  const u32 dists[] = {0u, 1u, 5000u, 2147483348u, 2147483647u};
  const int seeds[] = {11, 0, 5, -1};
  for (const Set &S : sets)
    for (u32 d : dists)
      for (int seed : seeds) {
        if (&S == &sets[3] && !(d == 0u || d == 5000u)) continue;  // the big set at two distances
        std::vector<PpRecord> rec = random_set(g, S.n_uni, S.n_reads, S.max_cand, S.n_seq, S.base, S.span, S.hop);
        const size_t n = rec.size();
        std::vector<u8> want(n), got;
        orc_alloc_stats ws{}, gs{};
        std::vector<u32> weight, midx;
        const int orc_rc = orc_allocate_flags((const orc_alloc_record *)rec.data(), n, (u32)S.n_seq, (int32_t)d, seed, want.data(), &ws);
        check(orc_rc == 0, "oracle found multi-mappings", orc_rc, 0);
        device_flow(rec, d, seed, got, gs, weight, midx);
        // every weight against the interval tree
        std::vector<OrcIntervalTree> trees((size_t)S.n_seq);
        for (const PpRecord &x : rec) if (pe_mapq(x) >= 4) { trees[x.w[1]].start.push_back(x.w[2]); trees[x.w[1]].end.push_back(x.w[2] + pe_len(x)); }
        for (auto &t : trees) t.build();
        for (size_t j = 0; j < midx.size(); ++j) {
          const PpRecord &x = rec[midx[j]];
          const u32 s = x.w[2], e = s + pe_len(x);
          const u32 c = trees[x.w[1]].count(s > d ? s - d : 0u, e + d);
          check(weight[j] == c, "weight", weight[j], c);
          wrapped_overlaps += e + d <= (s > d ? s - d : 0u) && c > 0;
          ++weights_checked;
        }
        check(memcmp(want.data(), got.data(), n) == 0, "keep flags", (long)std::count(got.begin(), got.end(), 1), (long)std::count(want.begin(), want.end(), 1));
        check(ws.n_multi == gs.n_multi, "n_multi", gs.n_multi, ws.n_multi);
        check(ws.n_allocated == gs.n_allocated, "n_allocated", gs.n_allocated, ws.n_allocated);
        check(ws.n_without_overlap == gs.n_without_overlap, "n_without_overlap", gs.n_without_overlap, ws.n_without_overlap);
        check(ws.n_draws == gs.n_draws, "n_draws", gs.n_draws, ws.n_draws);
        check(ws.n_uni_after == gs.n_uni_after && ws.n_multi_after == gs.n_multi_after, "is_unique split", gs.n_uni_after, ws.n_uni_after);
        if (&S == &sets[3]) check(gs.n_draws > 10000, "draws of the big set", gs.n_draws, 10000);
        ++cases;
      }
  printf("cases=%ld draws=%ld weights=%ld wrapped_overlaps=%ld bad=%ld\n", cases, draws_total, weights_checked, wrapped_overlaps, bad);
  return bad != 0;
}
'''


def test_allocation_kernels_and_draw_equal_the_restatement(tmp_path):
    main = MAIN.replace("ALLOC_ORACLE_H", os.path.join(HERE, "allocate_oracle.h"))
    out = emu.run(tmp_path, emu.PIPELINE + ["postprocess.cuh", "allocate.cuh"], main, timeout=1800)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["cases"]) >= 148 and int(f["draws"]) > 500000 and int(f["weights"]) > 100000 and int(f["wrapped_overlaps"]) > 100, out.stdout
