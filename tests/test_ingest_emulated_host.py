"""FASTQ parsing on the device (chromap_b200/csrc/ingest.cuh: newline flags, per-record spans / name spans / format checks, packing)
run UNCHANGED on the host emulation (tests/cta_emu.h) in cmx_ingest_fastq's sequence (a stream compaction and a prefix sum in
CUB's place) against the host reader with kseq's behaviour (csrc/host/seqio.cc, the reader the CLI falls back to): names,
bases and qualities of every record for LF and CRLF files, names with comments, reads of every length; and the reports on
input that is not plain 4-line FASTQ (a header without '@', a separator without '+', an empty read, quality and sequence of
different lengths) that send the caller to the host reader."""
import os

from tests import emu

MAIN = r'''
#include "%(seqio_h)s"
struct Parsed { u32 n = 0; std::vector<u32> off, spans; std::string seq, qual; IngestStats st; bool whole = true; };
static Parsed device_parse(const std::string &text) {
  Parsed P;
  const u32 nb = (u32)text.size();
  std::vector<u8> flag(nb + 1);
  emu_grid_serial((int)((nb + 255) / 256), 256, [&]() { newline_flag_kernel(text.data(), nb, flag.data()); });
  std::vector<u32> nl;
  for (u32 i = 0; i < nb; ++i) if (flag[i]) nl.push_back(i);           // DeviceSelect::Flagged over a counting iterator
  if (nl.size() %% 4 != 0) { P.whole = false; return P; }
  const u32 n = (u32)(nl.size() / 4);
  P.n = n;
  std::vector<u32> seq_start(n + 1), qual_start(n + 1), len(n + 1, 0);
  P.spans.assign((size_t)2 * n + 2, 0);
  P.st = IngestStats{0, 0, 0, 0, 0xFFFFFFFFu, 0};
  emu_grid_serial((int)((n + 255) / 256), 256, [&]() { ingest_record_kernel(text.data(), nl.data(), n, seq_start.data(), qual_start.data(), len.data(), P.spans.data(), &P.st); });
  P.off.assign(n + 1, 0);
  for (u32 i = 0; i < n; ++i) P.off[i + 1] = P.off[i] + len[i];         // DeviceScan::ExclusiveSum
  P.seq.assign((size_t)P.off[n] + 64, '?'); P.qual.assign((size_t)P.off[n] + 64, '?');
  emu_grid_serial((int)(((u64)n * 32 + 255) / 256), 256, [&]() { ingest_pack_kernel(text.data(), seq_start.data(), qual_start.data(), P.off.data(), nl.data(), n, &P.seq[0], &P.qual[0]); });
  return P;
}
int main(int argc, char **argv) {
  std::mt19937 g(103);
  long bad = 0, n_files = 0, n_records = 0, n_reported = 0;
  const std::string dir = argc > 1 ? argv[1] : "/tmp";
  for (int it = 0; it < 120; ++it) {
    const bool crlf = it %% 4 == 1;
    const int defect = it %% 3 == 2 ? 1 + (int)(g() %% 4) : 0;          // 1 header without '@', 2 separator without '+', 3 empty read, 4 short quality
    const int n = 1 + (int)(g() %% 300);
    const int hit = (int)(g() %% n);
    std::string text;
    auto eol = [&]() { if (crlf) text.push_back('\r'); text.push_back('\n'); };
    for (int r = 0; r < n; ++r) {
      const int L = defect == 3 && r == hit ? 0 : 1 + (int)(g() %% 160);
      text.push_back(defect == 1 && r == hit ? '>' : '@');
      text += "read" + std::to_string(r);
      if (g() %% 2) text += (g() %% 2 ? " 1:N:0:ACGT" : "\tcomment");
      eol();
      for (int i = 0; i < L; ++i) {   // bases, and one byte in eight beyond them: 0x80-0xFF, '.', IUPAC codes in both cases
        const u32 k = g() %% 8;
        text.push_back(k ? "ACGTNacgt"[g() %% 9] : g() %% 2 ? (char)(0x80 + g() %% 128) : ".RYKMSWBDHVnrykmswbdhv"[g() %% 22]);
      }
      eol();
      text += (defect == 2 && r == hit) ? "-" : (g() %% 2 ? "+" : "+read" + std::to_string(r));
      eol();
      const int QL = defect == 4 && r == hit ? std::max(0, L - 1 - (int)(g() %% 3)) : L;
      for (int i = 0; i < QL; ++i) text.push_back((char)(33 + g() %% 60));
      eol();
    }
    ++n_files;
    const Parsed P = device_parse(text);
    const bool reported = !P.whole || P.st.bad_header || P.st.bad_plus || P.st.empty_reads || P.st.qual_mismatch;
    if (defect) {
      ++n_reported;
      const bool right = (defect == 1 && P.st.bad_header == 1) || (defect == 2 && P.st.bad_plus == 1) || (defect == 3 && P.st.empty_reads >= 1) || (defect == 4 && P.st.qual_mismatch == 1);
      if (!reported || !right) { if (bad < 6) printf("DEFECT %%d not reported as such (it=%%d): header %%u plus %%u empty %%u qual %%u\n", defect, it, P.st.bad_header, P.st.bad_plus, P.st.empty_reads, P.st.qual_mismatch); ++bad; }
      continue;
    }
    const std::string path = dir + "/ingest.fq";
    FILE *f = fopen(path.c_str(), "wb"); fwrite(text.data(), 1, text.size(), f); fclose(f);
    cmxhost::SeqReader rd;
    rd.Open(path);
    std::string nm, sq, ql;
    bool ok = !reported && (int)P.n == n;
    u32 mn = 0xFFFFFFFFu, mx = 0;
    for (int r = 0; ok && r < n; ++r) {
      ok = rd.Next(&nm, &sq, &ql);
      if (!ok) break;
      const u32 o = P.off[r], l = P.off[r + 1] - o;
      ok = l == sq.size() && memcmp(P.seq.data() + o, sq.data(), l) == 0 && memcmp(P.qual.data() + o, ql.data(), l) == 0 && P.spans[2 * r + 1] == nm.size() &&
           memcmp(text.data() + P.spans[2 * r], nm.data(), nm.size()) == 0;
      mn = std::min(mn, l); mx = std::max(mx, l);
      ++n_records;
    }
    ok = ok && P.st.min_len == mn && P.st.max_len == mx && !rd.Next(&nm, &sq, &ql);
    if (!ok) { if (bad < 6) printf("PARSE it=%%d crlf=%%d records %%u / %%d\n", it, crlf, P.n, n); ++bad; }
  }
  printf("files=%%ld records=%%ld defective_files=%%ld bad=%%ld\n", n_files, n_records, n_reported, bad);
  return bad != 0;
}
'''


def test_fastq_ingest_kernels_equal_the_host_reader(tmp_path):
    host = os.path.join(emu.CSRC, "host")
    out = emu.run(tmp_path, ["device_common.cuh", "ingest.cuh"], MAIN % dict(seqio_h=os.path.join(host, "seqio.h")), args=[str(tmp_path)], timeout=1200,
                  sources=[os.path.join(host, "seqio.cc")], libs=["-lz"])
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["records"]) > 5000 and int(f["defective_files"]) > 20, out.stdout
