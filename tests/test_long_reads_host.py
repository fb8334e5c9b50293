"""The SAM path's banded semi-global aligner at its long instance (sam_band_align<SAM_MAX_L_LONG>, reads of 161 to 320
bases, chromap_b200/csrc/sam_kernels.cuh) compiled for the HOST against the oracle's restatement of ksw_semi_global3
(oracle_chromap.cc, pinned to the reference binary's SAM output of such reads by tests/test_oracle_long.py), on random windows
with substitutions, insertions, deletions, N's and every e the SAM path takes, as tests/test_sam_align_host.py does for the
instance of reads up to 160 bases."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "%(root)s/chromap_b200/csrc/sam_kernels.cuh"
extern "C" int orc_sg_align_test(const char *win, int wlen, const char *read, int rlen, int w, unsigned *cigar, int cap, int *start, int *end);
static unsigned code(char c) { switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; } }
int main() {
  srand(11);
  long bad = 0, n_indel = 0, tot = 0;
  for (int it = 0; it < 40000; ++it) {
    const int e = 1 + rand() %% 8, L = 161 + rand() %% 160;   // 161 .. 320: the long instance only
    std::string ref(L + 2 * e + 40, 'A');
    for (auto &c : ref) c = "ACGT"[rand() %% 4];
    if (rand() %% 10 == 0) for (int q = 0; q < 3; ++q) ref[rand() %% ref.size()] = 'N';
    if (rand() %% 8 == 0) for (auto &c : ref) c = "AC"[rand() %% 2];   // low complexity: many ties
    // read = a copy of ref[off .. off + L') with edits
    const int off = rand() %% (2 * e + 1);
    std::string read;
    int p = off;
    const int n_edit = rand() %% (e + 2);
    std::vector<int> at;
    for (int q = 0; q < n_edit; ++q) at.push_back(rand() %% L);
    while ((int)read.size() < L) {
      bool ed = false;
      for (int a : at) if (a == (int)read.size()) ed = true;
      if (ed) {
        const int k = rand() %% 3;
        if (k == 0) { read.push_back("ACGT"[rand() %% 4]); ++p; }
        else if (k == 1) { read.push_back("ACGT"[rand() %% 4]); ++n_indel; }
        else { ++p; read.push_back(ref[p %% ref.size()]); ++p; ++n_indel; }
      } else { read.push_back(ref[p %% ref.size()]); ++p; }
    }
    if (rand() %% 12 == 0) read[rand() %% L] = 'N';
    const int wlen = L + 2 * e;
    unsigned c1[64], c2[64];
    int s1 = -1, e1 = -1, s2 = -1, e2 = -1;
    const int n1 = orc_sg_align_test(ref.data(), wlen, read.data(), L, 2 * e + 1, c1, 24, &s1, &e1);
    const int n2 = sam_band_align<SAM_MAX_L_LONG>(L, e, 1, 4, 6, 1, 6, 1, [&](int j) { return code(ref[j]); }, [&](int i) { return code(read[i]); }, c2, 24, &s2, &e2);
    ++tot;
    const bool ovf1 = n1 > 24;
    if (ovf1) { if (n2 != -1) ++bad; continue; }
    if (n1 != n2 || s1 != s2 || e1 != e2 || memcmp(c1, c2, 4 * n1)) { if (bad < 5) printf("MISMATCH e=%%d L=%%d n %%d/%%d start %%d/%%d end %%d/%%d\n", e, L, n1, n2, s1, s2, e1, e2); ++bad; }
  }
  printf("windows=%%ld bad=%%ld edits_with_indels=%%ld\n", tot, bad, n_indel);
  return bad != 0;
}
'''


def test_long_sam_band_align_equals_the_oracles_ksw_restatement(tmp_path):
    src = tmp_path / "t.cc"
    src.write_text(SRC % dict(root=ROOT))
    exe = tmp_path / "t"
    lib = os.path.join(ROOT, "oracle", "liboracle.so")
    assert os.path.exists(lib), "oracle/liboracle.so not built (__graft_entry__.build())"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(src), lib, "-Wl,-rpath," + os.path.dirname(lib), "-fopenmp"])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-800:]
    n_windows, n_indels = (int(f.split("=")[1]) for f in out.stdout.split()[::2])
    assert n_windows == 40000 and n_indels > 10000, out.stdout
