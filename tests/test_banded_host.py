"""The banded bit-vector aligners of the CUDA path (chromap_b200/csrc/pipeline_kernels.cuh: three-bit-plane pattern window,
software-pipelined `banded_align`, `banded_traceback` with its Hamming shortcut, the two drop-off aligners of the split path
folded into one `banded_align_dropoff`) compiled for the HOST and compared with the oracle's restatements of alignment.cc
(pinned to the reference binary by tests/test_oracle_golden.py) on random windows: substitutions, indels, N's, soft-masked
reference bases, chimeric reads, every e the path accepts.  The same comparison runs on the GPU in the stage tests; this one
keeps the device formulation honest on machines without one.  A second run feeds the steps that compare raw bytes — the Hamming
shortcut of `banded_traceback` and the Hi-C gap extension `adjust_gap_beginning` (signed chars, `b - 'a' + 'A'`) — bytes beyond
upper-case ACGTN and counts the inputs on which a case-folded or unsigned compare would give another answer."""
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


RAW_BYTES_MAIN = r"""
extern "C" void orc_banded_traceback(int e, int min_errors, const char *pattern, const char *text, int read_len, int *start_pos);
extern "C" int orc_banded_align(int e, const char *pattern, const char *text, int read_len, int *end_pos);
extern "C" int orc_adjust_gap_beginning(int strand, const char *ref, const char *read, int *gap, int read_end, int ref_start, int ref_end);
static const char kNoBase[] = "NnRYKMSWBDHVrykmswbdhv.";   // bytes CharToUint8 maps to 4 (with the high and control bytes)
static char no_base() { const int k = rand() % 4; return k == 0 ? (char)(0x80 + rand() % 128) : k == 1 ? (char)(1 + rand() % 31) : kNoBase[rand() % (sizeof(kNoBase) - 1)]; }
static char flip_case(char c) { return c >= 'a' && c <= 'z' ? (char)(c - 32) : c >= 'A' && c <= 'Z' ? (char)(c + 32) : c; }
// the gap extension with unsigned bytes: what a compare on u8 would give (counted, not asserted)
static int gap_unsigned(int strand, const u8 *ref, const u8 *read, int *gap, int read_end, int ref_start, int ref_end) {
  int i, j;
  if (strand == 0) {
    for (i = *gap - 1, j = ref_start - 1; i >= 0 && j >= 0; --i, --j) if (read[i] != ref[j] && read[i] != ref[j] - 'a' + 'A') break;
    *gap = i + 1;
    return j + 1;
  }
  for (i = read_end + 1, j = ref_end + 1; read[i] && ref[j]; ++i, ++j) if (read[i] != ref[j] && read[i] != ref[j] - 'a' + 'A') break;
  *gap = *gap + i - (read_end + 1);
  return j - 1;
}
int main() {
  srand(41);
  long bad = 0, n_tb = 0, n_raw_ne_folded = 0, n_folded_differs = 0, n_gap = 0, n_gap_alt = 0, n_gap_signed = 0;
  // ---- the Hamming shortcut of banded_traceback: raw bytes, where a case fold would count fewer mismatches
  for (int it = 0; it < 300000; ++it) {
    const int e = 1 + rand() % 8, L = 25 + rand() % 136;
    std::string ref(L + 2 * e + 64, 'A');
    const char *alpha = rand() % 3 == 0 ? "AC" : rand() % 2 ? "AAAC" : "ACGT";   // low-complexity windows: ties between starts
    for (auto &c : ref) c = alpha[rand() % strlen(alpha)];
    for (int q = rand() % 4; q > 0; --q) ref[rand() % ref.size()] = no_base();
    if (rand() % 2) { const int at = rand() % (int)ref.size(), ln = 1 + rand() % 40; for (int i = at; i < std::min((int)ref.size(), at + ln); ++i) ref[i] = flip_case(ref[i]); }
    const int off = e + rand() % 3 - 1;
    std::string read = ref.substr((size_t)off, (size_t)L);
    for (int q = rand() % (e + 2); q > 0; --q) {   // substitutions and single-base indels
      const int p = rand() % L, k = rand() % 3;
      if (k == 0) read[p] = "ACGT"[rand() % 4];
      else if (k == 1) { read.erase((size_t)p, 1); read.push_back("ACGT"[rand() % 4]); }
      else { read.insert((size_t)p, 1, "ACGT"[rand() % 4]); read.resize((size_t)L); }
    }
    for (auto &c : read) {   // a byte that is no base opposite another one; lower case, or upper case opposite soft-masking
      if (!strchr("ACGTacgt", c) && rand() % 2) c = no_base();
      if (rand() % 6 == 0) c = flip_case(c);
    }
    if (rand() % 5 == 0) for (auto &c : read) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    int ep = -7;
    const int r1 = orc_banded_align(e, ref.data(), read.data(), L, &ep);
    if (r1 > e || r1 == 0) continue;
    const int vws = ep + 1 - L - e;
    if (vws < 0 || vws + L + 2 * e > (int)ref.size()) continue;
    int s1 = -9;
    orc_banded_traceback(e, r1, ref.data() + vws, read.data(), L, &s1);
    const int s2 = banded_traceback(e, r1, L, [&](int i) { return (u8)ref[vws + i]; }, [&](int i) { return (u8)read[i]; });
    ++n_tb;
    int raw = 0, folded = 0;
    for (int i = 0; i < L; ++i) { raw += ref[vws + e + i] != read[i]; folded += base_code((u8)ref[vws + e + i]) != base_code((u8)read[i]); }
    n_raw_ne_folded += raw != folded;
    n_folded_differs += raw != r1 && folded == r1 && s1 != e;   // a shortcut on folded bytes would return e here
    if (s1 != s2) { if (bad < 5) printf("TRACEBACK e=%d L=%d min_err=%d start %d/%d\n", e, L, r1, s1, s2); ++bad; }
  }
  // ---- adjust_gap_beginning: read bytes against reference bytes of every kind, both strands
  for (int it = 0; it < 300000; ++it) {
    const int n = 200 + rand() % 200;
    std::string ref((size_t)n + 64, '\0');   // NUL padded after the sequence, as the library lays the reference out
    for (int i = 0; i < n; ++i) {
      const int k = rand() % 10;
      ref[i] = k < 5 ? "ACGT"[rand() % 4] : k < 8 ? "acgtn"[rand() % 5] : k == 8 ? (char)(0x80 + rand() % 128) : (char)(1 + rand() % 31);
    }
    const int strand = rand() % 2, full = 60 + rand() % 100, gap0 = 1 + rand() % 40, read_end = full - 1 - (strand ? gap0 : 0);
    const int ref_start = 50 + rand() % (n - 150), ref_end = ref_start + 40;
    std::string read((size_t)full + 1, '\0');
    for (int i = 0; i < full; ++i) {   // opposite the reference as the extension walks it: equal, 32 lower (the signed rule), case-folded or other
      const int j = strand == 0 ? ref_start - gap0 + i : ref_end + 1 + (i - read_end - 1);
      const u8 b = j >= 0 && j < n ? (u8)ref[j] : (u8)'A';
      const int k = rand() % 12;
      read[i] = k < 6 ? (char)b : k < 9 ? (char)(u8)(b - 32) : k < 10 ? flip_case((char)b) : "ACGT"[rand() % 4];
      if (read[i] == 0) read[i] = 'A';
    }
    int g1 = gap0, g2 = gap0, g3 = gap0;
    const int a1 = orc_adjust_gap_beginning(strand, ref.data(), read.data(), &g1, read_end, ref_start, ref_end);
    const int a2 = adjust_gap_beginning(strand, (const u8 *)ref.data(), [&](int i) { return i < full ? (u8)read[i] : (u8)0; }, &g2, read_end, ref_start, ref_end);
    const int a3 = gap_unsigned(strand, (const u8 *)ref.data(), (const u8 *)read.data(), &g3, read_end, ref_start, ref_end);
    ++n_gap;
    n_gap_signed += a3 != a1 || g3 != g1;
    {   // did the extension step over a byte that matched only through b - 'a' + 'A' (a lower-case or high reference byte)?
      const int steps = strand == 0 ? gap0 - g1 : g1 - gap0;
      for (int t = 0; t < steps; ++t) {
        const int i = strand == 0 ? gap0 - 1 - t : read_end + 1 + t, j = strand == 0 ? ref_start - 1 - t : ref_end + 1 + t;
        if (read[i] != ref[j]) { ++n_gap_alt; break; }
      }
    }
    if (a1 != a2 || g1 != g2) { if (bad < 10) printf("GAP strand=%d gap %d: ref %d/%d gap %d/%d\n", strand, gap0, a1, a2, g1, g2); ++bad; }
  }
  printf("tracebacks=%ld raw_ne_folded=%ld folded_differs=%ld gaps=%ld gap_alt=%ld gap_signed=%ld bad=%ld\n", n_tb, n_raw_ne_folded, n_folded_differs, n_gap,
         n_gap_alt, n_gap_signed, bad);
  return bad != 0;
}
"""


def test_raw_byte_compares_equal_the_oracle(tmp_path):
    """banded_traceback's Hamming shortcut and adjust_gap_beginning on bytes beyond upper-case ACGTN: lower case opposite upper
    case, bytes that are no base (N, n, '.', IUPAC codes, control and high bytes) opposite each other, read bytes 32 below the
    reference byte.  Against the oracle's restatements; floors on the inputs where a case-folded shortcut or an unsigned compare
    would have answered differently, so that a device formulation with either slip fails here."""
    out = emu.run(tmp_path, emu.PIPELINE, RAW_BYTES_MAIN, timeout=900)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-1200:]
    f = {k: int(v) for k, v in (kv.split("=") for kv in out.stdout.split() if "=" in kv)}
    assert f["tracebacks"] > 50000 and f["raw_ne_folded"] > 10000 and f["gaps"] == 300000, out.stdout
    # about half of the first run: 175,854 extensions stepped over a byte that matched only through b - 'a' + 'A', and on 40,613
    # an unsigned compare would have stopped elsewhere.  (folded_differs: tracebacks whose start a case-folded shortcut would change;
    # none has been found, see the README.)
    assert f["gap_alt"] > 85000 and f["gap_signed"] > 20000, out.stdout
