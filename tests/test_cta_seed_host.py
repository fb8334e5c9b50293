"""The block-cooperative building blocks of the overflow tiers' seeding kernel (chromap_b200/csrc/pipeline_kernels.cuh) run
UNCHANGED on the host emulation of a CTA (tests/cta_emu.h):
  * `cta_sort_keys` / `cta_sort_pairs` (hybrid shared/global bitonic sorts) against std::sort,
  * `cta_cluster` (streamed) and `cta_cluster_par` (segment-parallel) against the sequential clustering scan `cluster_hits`
    (candidate_processor.cc:283-342; the form the tier-0 kernel uses and the GPU stage tests pin to the oracle),
  * `cta_minimizers` (k-mer hashes in parallel, window logic replayed over the seeds; fallback for even k / unusual w / N)
    against the oracle's `orc_minimizers` (minimizer_generator.cc:7-139)."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
extern "C" int orc_minimizers(const char *seq, u32 len, u32 seq_index, int k, int w, u64 *hash, u64 *hit, int cap);
int main() {
  std::mt19937 g(41);
  long bad = 0, n_sort = 0, n_pairs = 0, n_cluster = 0, n_mini = 0, n_fallback = 0;
  // ---- sorts
  const int NS[8] = {0, 1, 2, 37, 1000, 1024, 2500, 5000}, SMC[3] = {256, 1024, 4096}, NTS[3] = {32, 128, 512};
  for (int a = 0; a < 8; ++a) for (int b = 0; b < 3; ++b) {
    const int c = (a + b) %% 3;   // block sizes rotate over the (n, shared-memory) grid
    const int n = NS[a], sm_cap = SMC[b], nt = NTS[c];
    int np2 = 1; while (np2 < n) np2 <<= 1;
    std::vector<u64> v((size_t)np2 + 1), sm((size_t)sm_cap);
    for (int i = 0; i < n; ++i) v[i] = ((u64)g() << 32 | g()) >> (g() %% 3 ? 0 : 40);   // many duplicates in one third of the keys
    std::vector<u64> want(v.begin(), v.begin() + n);
    std::sort(want.begin(), want.end());
    emu_launch(nt, [&]() { cta_sort_keys(v.data(), n, sm.data(), sm_cap); });
    ++n_sort;
    for (int i = 0; i < n; ++i) if (v[i] != want[i]) { if (bad < 5) printf("SORT n=%%d sm=%%d nt=%%d at %%d\n", n, sm_cap, nt, i); ++bad; break; }
    // (key, tag) pairs: candidates by count descending, position ascending (candidate.h:23-33)
    std::vector<u64> pk((size_t)np2 + 1), smk((size_t)sm_cap);
    std::vector<u8> pt((size_t)np2 + 1), smt((size_t)sm_cap);
    std::vector<std::pair<u64, u8>> pw;
    for (int i = 0; i < n; ++i) { pk[i] = g() %% 5000; pt[i] = (u8)(1 + g() %% 6); pw.push_back({pk[i], pt[i]}); }
    auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };
    std::sort(pw.begin(), pw.end(), [&](const std::pair<u64, u8> &x, const std::pair<u64, u8> &y) { return cless(x.first, x.second, y.first, y.second); });
    emu_launch(nt, [&]() { cta_sort_pairs<u8>(pk.data(), pt.data(), n, ~0ull, (u8)0, cless, smk.data(), smt.data(), sm_cap); });
    ++n_pairs;
    for (int i = 0; i < n; ++i) if (pk[i] != pw[i].first || pt[i] != pw[i].second) { if (bad < 5) printf("PAIRS n=%%d sm=%%d nt=%%d at %%d\n", n, sm_cap, nt, i); ++bad; break; }
  }
  // ---- clustering
  for (int it = 0; it < 54; ++it) {
    const int nt = NTS[it %% 3], e = 1 + (int)(g() %% 12), need = 1 + (int)(g() %% 2);
    const int nh = (int)(g() %% (it %% 4 == 0 ? 5000 : 600));
    const u32 n_mm = 1 + g() %% 30;
    std::vector<u64> hits((size_t)nh);
    u64 p = 0;
    for (auto &h : hits) {                       // runs of nearby hits (clusters), repeated positions, several sequences
      const int m = (int)(g() %% 10);
      if (m == 0) p += 1000 + g() %% 100000; else if (m < 4) p += g() %% (2 * e + 2); else if (m < 8) p += 0; else p += 1 + g() %% 3;
      if (g() %% 200 == 0) p = ((p >> 32) + 1) << 32;
      h = p;
    }
    const int cap = 8192, sm_cap = it %% 2 ? 1024 : 4096;
    std::vector<u64> w_p((size_t)cap), a_p((size_t)cap), b_p((size_t)cap), sm((size_t)sm_cap);
    std::vector<u8> w_c((size_t)cap), a_c((size_t)cap), b_c((size_t)cap), aux((size_t)3 * sm_cap);
    const int want = cluster_hits(e, need, n_mm, hits.data(), nh, w_p.data(), w_c.data(), cap);
    int got_a = -1, got_b = -1, s_ret = 0, s_ret2 = 0;
    emu_launch(nt, [&]() { const int r = cta_cluster(e, need, n_mm, hits.data(), nh, a_p.data(), a_c.data(), cap, sm.data(), sm_cap, &s_ret); if (threadIdx.x == 0) got_a = r; });
    emu_launch(nt, [&]() { const int r = cta_cluster_par(e, need, n_mm, hits.data(), nh, b_p.data(), b_c.data(), cap, sm.data(), sm_cap, aux.data(), &s_ret2); if (threadIdx.x == 0) got_b = r; });
    ++n_cluster;
    bool ok = got_a == want && got_b == want;
    for (int i = 0; ok && i < want && i < cap; ++i) ok = w_p[i] == a_p[i] && w_c[i] == a_c[i] && w_p[i] == b_p[i] && w_c[i] == b_c[i];
    if (!ok) { if (bad < 5) printf("CLUSTER it=%%d nt=%%d e=%%d need=%%d nh=%%d n %%d/%%d/%%d\n", it, nt, e, need, nh, want, got_a, got_b); ++bad; }
  }
  // ---- minimizers of a long read by the CTA
  const int KW[6][2] = {{17, 7}, {21, 10}, {15, 11}, {16, 7}, {17, 5}, {19, 7}};
  for (int it = 0; it < 54; ++it) {
    const int k = KW[it %% 6][0], w = KW[it %% 6][1];
    const int len = 30 + (int)(g() %% 900);
    std::string r((size_t)len, 'A');
    const int mode = (int)(g() %% 5);
    for (int i = 0; i < len; ++i) r[i] = mode == 0 ? "AC"[g() %% 2] : mode == 1 ? "ACGT"[(i / (1 + it %% 4)) %% 4] : "ACGT"[g() %% 4];
    if (mode == 3) for (int q = 0; q < 3; ++q) r[g() %% len] = 'N';
    if (mode == 4) for (auto &ch : r) if (g() %% 3 == 0) ch = (char)tolower(ch);
    const int cap = 2048;
    std::vector<u64> wh((size_t)cap), whit((size_t)cap), gh((size_t)cap), work((size_t)len * 2 + 64);
    std::vector<u32> gp((size_t)cap);
    const int want = orc_minimizers(r.data(), (u32)len, 0, k, w, wh.data(), whit.data(), cap);
    int got = -1, s_flag = 0;
    emu_launch(128, [&]() { const int n = cta_minimizers((const u8 *)r.data(), len, k, w, gh.data(), gp.data(), cap, work.data(), &s_flag); if (threadIdx.x == 0) got = n; });
    ++n_mini;
    if (!((k & 1) && (w == 7 || w == 10 || w == 11)) || mode == 3) ++n_fallback;
    bool ok = got == want;
    for (int i = 0; ok && i < want; ++i) ok = gh[i] == wh[i] && (u64)gp[i] == (whit[i] & 0xFFFFFFFFull);
    if (!ok) { if (bad < 5) printf("MINIMIZERS it=%%d k=%%d w=%%d len=%%d mode=%%d n %%d/%%d\n", it, k, w, len, mode, got, want); ++bad; }
  }
  printf("sorts=%%ld pair_sorts=%%ld clusterings=%%ld minimizer_reads=%%ld fallback_reads=%%ld bad=%%ld\n", n_sort, n_pairs, n_cluster, n_mini, n_fallback, bad);
  return bad != 0;
}
'''


def test_cta_sorts_clustering_and_minimizers(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"))
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-1500:] + out.stderr[-800:]
