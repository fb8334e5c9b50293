"""The banded bit-vector aligners of the CUDA path (chromap_b200/csrc/pipeline_kernels.cuh: three-bit-plane pattern window,
software-pipelined `banded_align`, `banded_traceback` with its Hamming shortcut, the two drop-off aligners of the split path
folded into one `banded_align_dropoff`) compiled for the HOST and compared with the oracle's restatements of alignment.cc
(pinned to the reference binary by tests/test_oracle_golden.py) on random windows: substitutions, indels, N's, soft-masked
reference bases, chimeric reads, every e the path accepts.  The same comparison runs on the GPU in the stage tests; this one
keeps the device formulation honest on machines without one."""
from tests import emu

MAIN = r'''
extern "C" int orc_banded_align(int e, const char *pattern, const char *text, int read_len, int *end_pos);
extern "C" void orc_banded_traceback(int e, int min_errors, const char *pattern, const char *text, int read_len, int *start_pos);
extern "C" int orc_align_dropoff(int e, const char *pattern, const char *text, int read_len, int from_3_end, int *end_pos, int *read_len_out);
static std::string mutate(const std::string &ref, int off, int L, int n_edit, bool chimera) {
  std::string read;
  int p = off;
  std::vector<int> at;
  for (int q = 0; q < n_edit; ++q) at.push_back(rand() % L);
  const int cut = chimera ? 20 + rand() % (L > 40 ? L - 40 : 1) : L + 1;
  while ((int)read.size() < L) {
    if ((int)read.size() >= cut) { read.push_back("ACGT"[rand() % 4]); continue; }   // the far side of a ligation junction
    bool ed = false;
    for (int a : at) if (a == (int)read.size()) ed = true;
    if (ed) {
      const int k = rand() % 3;
      if (k == 0) { read.push_back("ACGT"[rand() % 4]); ++p; }
      else if (k == 1) read.push_back("ACGT"[rand() % 4]);
      else { ++p; read.push_back(ref[p % ref.size()]); ++p; }
    } else { read.push_back(ref[p % ref.size()]); ++p; }
  }
  return read;
}
int main() {
  srand(23);
  long bad = 0, n_align = 0, n_tb = 0, n_drop = 0, n_dp = 0, n_long = 0, n_long_tb = 0, n_long_drop = 0;
  for (int it = 0; it < 200000; ++it) {
    // one window in eight from a read beyond 164 bases: up to 4 x 832 (the last overflow tier's reads) and a little over
    const bool long_read = rand() % 8 == 0;
    const int e = 1 + rand() % 15, L = long_read ? 165 + rand() % 3236 : 25 + rand() % 140;
    n_long += long_read;
    std::string ref(L + 2 * e + 64, 'A');
    for (auto &c : ref) c = "ACGT"[rand() % 4];
    if (rand() % 8 == 0) for (auto &c : ref) c = "AC"[rand() % 2];
    if (rand() % 10 == 0) for (int q = 0; q < 3; ++q) ref[rand() % ref.size()] = 'N';
    if (rand() % 6 == 0) for (auto &c : ref) if (rand() % 3 == 0) c = (char)tolower(c);   // soft-masked stretches: the Hamming shortcut compares raw chars
    std::string read = mutate(ref, e + (rand() % 3 - 1), L, rand() % (e + 3), false);
    if (rand() % 12 == 0) read[rand() % L] = 'N';
    // ---- banded_align (alignment.cc:141-192)
    int ep1 = -7, ep2 = -7;
    const int r1 = orc_banded_align(e, ref.data(), read.data(), L, &ep1);
    const int r2 = banded_align(e, L, [&](int i) { return base_code((u8)ref[i]); }, [&](int i) { return base_code((u8)read[i]); }, &ep2);
    ++n_align;
    if (r1 != r2 || (r1 <= e && ep1 != ep2)) { if (bad < 5) printf("ALIGN e=%d L=%d err %d/%d end %d/%d\n", e, L, r1, r2, ep1, ep2); ++bad; }
    // ---- banded_traceback (alignment.cc:656-718) on the window the emit kernels hand it: ends at the mapping's end position
    if (r1 <= e) {
      const int vws = ep1 + 1 - L - e;           // verification window of the emit kernels (mapping_generator.h:696-711): it ends e past the mapping's end
      if (vws >= 0 && vws + L + 2 * e <= (int)ref.size()) {
        int s1 = -9;
        orc_banded_traceback(e, r1, ref.data() + vws, read.data(), L, &s1);
        const int s2 = banded_traceback(e, r1, L, [&](int i) { return (u8)ref[vws + i]; }, [&](int i) { return (u8)read[i]; });
        ++n_tb;
        n_long_tb += long_read;
        int ham = 0;
        for (int i = 0; i < L; ++i) ham += ref[vws + e + i] != read[i];
        if (r1 != 0 && ham != r1) ++n_dp;
        if (s1 != s2) { if (bad < 5) printf("TRACEBACK e=%d L=%d min_err=%d start %d/%d\n", e, L, r1, s1, s2); ++bad; }
      }
    }
    // ---- the drop-off aligners of the split path (alignment.cc:197-283, :285-376), e as the Hi-C preset and around it
    if (e <= 8 && L >= 40) {
      const std::string chim = mutate(ref, e, L, rand() % (e + 2), rand() % 2);
      for (int from3 = 0; from3 < 2; ++from3) {
        std::string txt = chim;
        if (from3) { std::string t2(txt.rbegin(), txt.rend()); txt = t2; }   // any text will do: both sides see the same one
        int a1 = 0, b1 = 0, a2 = 0, b2 = 0;
        const int d1 = orc_align_dropoff(e, ref.data(), txt.data(), L, from3, &a1, &b1);
        const int d2 = banded_align_dropoff(e, L, from3 != 0, [&](int i) { return base_code((u8)ref[i]); }, [&](int i) { return base_code((u8)txt[i]); }, &a2, &b2);
        ++n_drop;
        n_long_drop += long_read;
        if (d1 != d2 || a1 != a2 || b1 != b2) { if (bad < 5) printf("DROPOFF e=%d L=%d from3=%d err %d/%d end %d/%d len %d/%d\n", e, L, from3, d1, d2, a1, a2, b1, b2); ++bad; }
      }
    }
  }
  printf("aligned=%ld tracebacks=%ld (bit-vector path %ld) dropoffs=%ld long=%ld long_tracebacks=%ld long_dropoffs=%ld bad=%ld\n", n_align, n_tb, n_dp, n_drop, n_long,
         n_long_tb, n_long_drop, bad);
  return bad != 0;
}
'''


def test_device_banded_aligners_equal_the_oracle(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN, timeout=900)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-1200:]
    # the interesting branches were really taken
    f = dict(kv.split("=") for kv in out.stdout.replace("(bit-vector path ", "dp=").replace(")", "").split() if "=" in kv)
    assert int(f["dp"]) > 1000 and int(f["tracebacks"]) - int(f["dp"]) > 10000 and int(f["dropoffs"]) > 10000, out.stdout
    assert int(f["long"]) > 20000 and int(f["long_tracebacks"]) > 5000 and int(f["long_dropoffs"]) > 5000, out.stdout
