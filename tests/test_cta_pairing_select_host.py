"""Pairing and multi-mapper sampling of the CUDA path on the host emulation of a CTA (tests/cta_emu.h), kernels run UNCHANGED:
  * `pairing_kernel` (tier 0: sort + the reference's two-pointer sweep) and `pairing_cta_kernel` (overflow tiers: cooperative
    sort, the window of every mate-1 mapping by two binary searches, tallies merged by reduction) against the oracle's
    `pair_dir` (mapping_generator.h:346-484; pinned to the reference binary by tests/test_oracle_golden.py);
  * `select_kernel` (a warp advances std::mt19937(11) 624 outputs at a time and replays the reservoir sampling with libstdc++'s
    Lemire uniform_int_distribution, 32 draws per step) against std::mt19937 + std::uniform_int_distribution themselves — the
    reference's own generator (mapping_generator.h:199-214, chromap.h:863)."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <random>
extern "C" void orc_pair_stats_test(int e, int max_insert_size, int min_read_length, u32 L1, u32 L2, const int *n_map, const u64 *pos, const short *err, int *stats);
int main() {
  std::mt19937 g(61);
  long bad = 0, n_pairs = 0, with_best = 0, n_sel = 0, sampled = 0, rejections = 0;
  // ---- pairing
  for (int it = 0; it < 70; ++it) {
    const int e = it %% 2 ? 8 : 4, mc = 512;
    DevParams P{};
    P.e = e; P.max_insert = it %% 3 ? 2000 : 1000; P.min_read_len = 30; P.drop_rep = 500000; P.max_best = 1;
    const u32 L1 = 40 + g() %% 100, L2 = 40 + g() %% 100;
    int n_map[4];
    std::vector<u64> pos; std::vector<short> err;
    const u64 base = ((u64)(g() %% 2) << 32) | 100000u;
    for (int q = 0; q < 4; ++q) {
      n_map[q] = it %% 11 == 0 ? 0 : (int)(g() %% (it %% 5 == 0 ? 400 : 12));
      if (it %% 11 == 0 && (q == 0 || q == 3)) n_map[q] = 1 + (int)(g() %% 3);
      for (int i = 0; i < n_map[q]; ++i) {
        // clustered around a few loci so that windows hold several partners; repeated positions with different errors
        const u64 locus = base + (u64)(g() %% 6) * 1500;
        pos.push_back(locus + g() %% 700 + ((g() %% 16 == 0) ? (1ull << 32) : 0));
        err.push_back((short)(g() %% (e + 1)));
      }
    }
    pos.push_back(0); err.push_back(0);
    int want[4];
    orc_pair_stats_test(e, P.max_insert, P.min_read_len, L1, L2, n_map, pos.data(), err.data(), want);
    for (int form = 0; form < 2; ++form) {
      Scratch S{};
      S.caps = Caps{160, 64, 64, mc}; S.n_slots = 1;
      std::vector<ReadMeta> rmeta(2); std::vector<PairMeta> pmeta(1);
      std::vector<u64> map_pos((size_t)2 * 2 * mc); std::vector<short> map_err((size_t)2 * 2 * mc);
      S.rmeta = rmeta.data(); S.pmeta = pmeta.data(); S.map_pos = map_pos.data(); S.map_err = map_err.data();
      rmeta[0].len = (int)L1; rmeta[1].len = (int)L2;
      size_t o = 0;
      for (int q = 0; q < 4; ++q) {
        const int m = q >> 1, s = q & 1;
        rmeta[m].n_map[s] = n_map[q];
        for (int i = 0; i < n_map[q]; ++i, ++o) { map_pos[((size_t)m * 2 + s) * mc + i] = pos[o]; map_err[((size_t)m * 2 + s) * mc + i] = err[o]; }
      }
      int nbest = -1;
      if (form == 0) emu_launch(32, [&]() { pairing_kernel(P, S, &nbest); });
      else {
        const int sm_cap = 1024;
        std::vector<u64> dyn((size_t)sm_cap + sm_cap / 4 + 8);
        g_dyn_smem = dyn.data();
        emu_launch(128, [&]() { pairing_cta_kernel(P, S, &nbest, sm_cap); });
      }
      ++n_pairs;
      const bool none = n_map[0] + n_map[1] == 0 || n_map[2] + n_map[3] == 0;
      bool ok;
      if (none) ok = pmeta[0].status == ST_DROP && nbest == 0;
      else ok = pmeta[0].min_sum == want[0] && pmeta[0].n_best == want[1] && pmeta[0].second_min_sum == want[2] && pmeta[0].n_second_best == want[3] && nbest == want[1];
      if (!none && want[1] > 0) ++with_best;
      if (!ok) { if (bad < 6) printf("PAIRING it=%%d form=%%d got %%d,%%d,%%d,%%d want %%d,%%d,%%d,%%d\n", it, form, pmeta[0].min_sum, pmeta[0].n_best, pmeta[0].second_min_sum, pmeta[0].n_second_best, want[0], want[1], want[2], want[3]); ++bad; }
    }
  }
  // ---- multi-mapper sampling
  u32 mt_init[624];
  mt_init_fill(mt_init);
  for (int it = 0; it < 12; ++it) {
    DevParams P{};
    P.max_best = 1 + (int)(g() %% 8); P.se = it %% 10 == 9;
    const int mb = P.max_best;
    const int n_chunks = 1 + (int)(g() %% 4);
    std::vector<int> chunk_start{0};
    for (int c = 0; c < n_chunks; ++c) chunk_start.push_back(chunk_start.back() + 1 + (int)(g() %% 150));
    const int n = chunk_start.back();
    std::vector<int> nbest((size_t)n), sel((size_t)n * mb, -1), want((size_t)n * mb);
    for (auto &x : nbest) { const int m = (int)(g() %% 10); x = m < 6 ? (int)(g() %% (mb + 1)) : m < 9 ? mb + 1 + (int)(g() %% 40) : mb + 1 + (int)(g() %% 3000); }
    for (int c = 0; c < n_chunks; ++c) {
      std::mt19937 gen(11);
      for (int p = chunk_start[c]; p < chunk_start[c + 1]; ++p) {
        int *s_ = &want[(size_t)p * mb];
        for (int j = 0; j < mb; ++j) s_[j] = j;
        if (nbest[p] > mb) {
          if (P.se) gen.seed(11);
          for (int i = mb; i < nbest[p]; ++i) { std::uniform_int_distribution<int> dist(0, i); const int j = dist(gen); if (j < mb) s_[j] = i; }
          std::sort(s_, s_ + mb);
          ++sampled;
        }
      }
    }
    emu_launch(128, [&]() { select_kernel(P, n_chunks, chunk_start.data(), nbest.data(), sel.data(), mt_init); });
    ++n_sel;
    if (sel != want) {
      if (bad < 6) { int q = 0; while (sel[q] == want[q]) ++q; printf("SELECT it=%%d mb=%%d se=%%d first difference at pair %%d slot %%d: %%d / %%d (nbest %%d)\n", it, mb, P.se, q / mb, q %% mb, sel[q], want[q], nbest[q / mb]); }
      ++bad;
    }
  }
  printf("pairings=%%ld with_best=%%ld selections=%%ld sampled_pairs=%%ld bad=%%ld\n", n_pairs, with_best, n_sel, sampled, bad);
  (void)rejections;
  return bad != 0;
}
'''


def test_pairing_kernels_and_multimapper_sampling(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"))
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2000:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["with_best"]) > 40 and int(f["sampled_pairs"]) > 300, out.stdout
