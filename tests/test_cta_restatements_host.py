"""The overflow tiers' exact parallel restatements of the reference's sequential candidate sweeps
(chromap_b200/csrc/cta_pair_candidates.cuh: `cta_merge_cands` = MergeCandidates, candidate_processor.cc:345-414;
`cta_pe_filter` = ReduceCandidatesForPairedEndReadOnOneDirection, :416-484) run UNCHANGED on a host emulation of a CTA
(tests/cta_emu.h: one OS thread per CUDA thread, pthread barriers, shuffles through a per-warp buffer) and compared element
for element with the sequential formulations the tier-0 kernels use (`merge_cands`, `pe_filter_dir` in pipeline_kernels.cuh,
which are the ones the GPU stage tests pin to the oracle).  Lists are random with many equal / near-equal positions, several
reference sequences, counts around the rule's thresholds; block sizes 32 .. 512 as the tiers launch them."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
static void gen(std::mt19937 &g, int n, int n_seq, u32 span, std::vector<u64> &p, std::vector<u8> &c) {
  p.resize(n); c.resize(n);
  for (int i = 0; i < n; ++i) p[i] = ((u64)(g() %% n_seq) << 32) | (u64)(g() %% span);
  std::sort(p.begin(), p.end());
  // candidate lists hold distinct positions (a cluster yields one candidate)
  p.erase(std::unique(p.begin(), p.end()), p.end());
  c.resize(p.size());
  for (auto &x : c) x = (u8)(1 + g() %% 12);
}
int main() {
  std::mt19937 g(17);
  long bad = 0, n_merge = 0, n_filter = 0, kept_unpaired = 0;
  const int NTS[5] = {32, 64, 128, 256, 512};
  for (int it = 0; it < 160; ++it) {
    const int nt = NTS[it %% 5], e = 1 + (int)(g() %% 12);
    const int n_seq = 1 + (int)(g() %% 3);
    const u32 span = 50 + g() %% 5000;
    std::vector<u64> p1, p2;
    std::vector<u8> c1, c2;
    gen(g, (int)(g() %% 700), n_seq, span, p1, c1);
    gen(g, (int)(g() %% 700), n_seq, span, p2, c2);
    if (it %% 7 == 0) { p1.clear(); c1.clear(); }
    if (it %% 11 == 0) { p2.clear(); c2.clear(); }
    const int n1 = (int)p1.size(), n2 = (int)p2.size(), cap = 4096;
    // ---- MergeCandidates
    {
      std::vector<u64> a = p1, po(cap), mp(n1 + n2 + 1), op(cap);
      std::vector<u8> ac = c1, co(cap), mc(n1 + n2 + 1), kf(n1 + n2 + 1), oc(cap);
      a.resize(cap); ac.resize(cap);
      const int want = merge_cands(e, a.data(), ac.data(), n1, p2.data(), c2.data(), n2, po.data(), co.data(), cap);
      int got = -1;
      int s_warp[32];
      emu_launch(nt, [&]() {
        const int r = cta_merge_cands(e, p1.data(), c1.data(), n1, p2.data(), c2.data(), n2, mp.data(), mc.data(), kf.data(), op.data(), oc.data(), cap, s_warp);
        if (threadIdx.x == 0) got = r;
      });
      ++n_merge;
      bool ok = got == want;
      for (int i = 0; ok && i < want; ++i) ok = a[i] == op[i] && ac[i] == oc[i];
      if (!ok) { if (bad < 5) printf("MERGE it=%%d nt=%%d e=%%d n1=%%d n2=%%d size %%d/%%d\n", it, nt, e, n1, n2, got, want); ++bad; }
    }
    // ---- paired-end filter
    {
      const u32 dist = 10 + g() %% 2000;
      std::vector<u64> f1p(n1 + 1), f2p(n2 + 1), o1p(n1 + 1), o2p(n2 + 1);
      std::vector<u8> f1c(n1 + 1), f2c(n2 + 1), o1c(n1 + 1), o2c(n2 + 1), fl1(n1 + 1), fl2(n2 + 1);
      int wa = 0, wb = 0, ga = -1, gb = -1;
      pe_filter_dir(dist, p1.data(), c1.data(), n1, p2.data(), c2.data(), n2, f1p.data(), f1c.data(), &wa, f2p.data(), f2c.data(), &wb);
      int s_warp[32];
      emu_launch(nt, [&]() {
        int a = 0, b = 0;
        cta_pe_filter(dist, p1.data(), c1.data(), n1, p2.data(), c2.data(), n2, o1p.data(), o1c.data(), &a, o2p.data(), o2c.data(), &b, fl1.data(), fl2.data(), s_warp);
        if (threadIdx.x == 0) { ga = a; gb = b; }
      });
      ++n_filter;
      bool ok = ga == wa && gb == wb;
      for (int i = 0; ok && i < wa; ++i) ok = f1p[i] == o1p[i] && f1c[i] == o1c[i];
      for (int i = 0; ok && i < wb; ++i) ok = f2p[i] == o2p[i] && f2c[i] == o2c[i];
      for (int i = 0; i < n1; ++i) kept_unpaired += fl1[i] == 2;
      if (!ok) { if (bad < 5) printf("FILTER it=%%d nt=%%d dist=%%u n1=%%d n2=%%d sizes %%d/%%d %%d/%%d\n", it, nt, dist, n1, n2, ga, wa, gb, wb); ++bad; }
    }
  }
  printf("merges=%%ld filters=%%ld unpaired_flagged=%%ld bad=%%ld\n", n_merge, n_filter, kept_unpaired, bad);
  return bad != 0;
}
'''


def test_cta_merge_and_pe_filter_equal_the_sequential_sweeps(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"), timeout=1200)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-1500:] + out.stderr[-500:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["unpaired_flagged"]) > 15, out.stdout   # the unpaired-candidate rule was exercised
