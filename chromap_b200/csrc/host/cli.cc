// chromap-b200 — command-line front end that keeps the reference's CLI for the supported path
// (chromap_driver.cc:16-159 option names, :247-275 presets, :451-531 checks): index construction (-i) on the
// GPU with the reference's index file format, and paired-end mapping to BED through the C ABI.
// Everything here is host plumbing around cmx_map_batch_pe; the batch loop replaces chromap.h:851-1290.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <algorithm>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../../include/chromap_b200.h"
#include <fcntl.h>
#include <glob.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

#include "seqio.h"

using cmxhost::IndexFile;
using cmxhost::IndexMap;
using cmxhost::Reference;
using cmxhost::SeqReader;

static void Die(const std::string &msg) {  // utils.h:71-74
  fprintf(stderr, "%s\n", msg.c_str());
  exit(255);
}
// --barcode-translate: the file's lines through zlib (plain or gzipped, as the reference's gzopen / gzgets), parsed before
// any device work so that a table the GPU path refuses needs no device.  A file that cannot be opened has no lines.
static void LoadBarcodeTranslation(const std::string &path, cmx_barcode_translation *tr) {
  std::string text;
  gzFile f = gzopen(path.c_str(), "r");
  if (f) {
    char buf[1 << 16];
    int got;
    while ((got = gzread(f, buf, sizeof(buf))) > 0) text.append(buf, (size_t)got);
    gzclose(f);
  }
  char err[256] = "";
  if (cmx_parse_barcode_translation(text.data(), text.size(), tr, err, sizeof(err)) != CMX_OK)
    Die("chromap-b200: --barcode-translate " + path + ": " + (f ? std::string(err) : "cannot be read") +
        "; the reference's result for such a table is undefined or an artifact of its reader, so the GPU path refuses it");
}
// Translate's failure (barcode_translator.h:87-91), without the partial output file the reference leaves behind
static void DieBarcodeNotTranslated(const std::string &detail) {
  fprintf(stderr, "Barcode does not exist in the translation table.\n");
  Die("chromap-b200: " + detail + "; no output was written");
}
template <class F> static void OpenReads(F *f, const std::string &path) {  // a SeqReader or a RawFile
  if (!f->Open(path)) Die("Cannot find sequence file " + path);
}
static double Now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Batch {
  std::string s1, s2;
  std::vector<uint32_t> o1{0}, o2{0};
  std::vector<std::string> names1;  // read-1 names, kept for pairs / SAM output only
  std::vector<std::string> names2;  // SAM only
  std::string q1, q2;               // qualities in the layout of s1 / s2 (SAM only)
  std::string bc, bq;               // cell barcodes + qualities, bc_len bytes per pair (scATAC)
  uint32_t n = 0;
  uint32_t max_len = 0;  // the longest read of either mate
  bool dev = false;      // reads were packed on the device (cmx_ingest_fastq): dev_in holds device pointers
  cmx_batch dev_in{};
  void Clear() { dev = false; s1.clear(); s2.clear(); o1.assign(1, 0); o2.assign(1, 0); names1.clear(); names2.clear(); q1.clear(); q2.clear(); bc.clear(); bq.clear(); n = 0; max_len = 0; }
};

// Raw text of one read file for the device-side FASTQ parser.  Plain files are read with read(2) straight into a page-locked
// buffer (no zlib copy, H2D at PCIe speed); gzip files go through gzread.  Whole 4-line records are cut off the front of the
// buffer (same rule as cmx_fastq_cut, but the scan remembers where it stopped instead of starting over after every refill),
// the rest stays for the next batch.
struct RawBuf {  // uninitialised page-aligned bytes (a std::vector would zero-fill hundreds of megabytes before they are read into)
  char *p = nullptr;
  size_t n = 0;
  char *data() { return p; }
  const char *data() const { return p; }
  size_t size() const { return n; }
  char &operator[](size_t i) { return p[i]; }
  void Grow(size_t bytes, size_t keep) {
    char *q = (char *)aligned_alloc(4096, (bytes + 4095) & ~(size_t)4095);
    if (!q) { fprintf(stderr, "chromap-b200: out of memory\n"); exit(255); }
    if (keep) memcpy(q, p, keep);
    free(p);
    p = q; n = bytes;
  }
  ~RawBuf() { free(p); }
};
struct RawFile {
  gzFile f = nullptr;
  int fd = -1;
  RawBuf buf;
  size_t have = 0;
  bool eof = false, pinned = false;
  size_t fpos = 0;                   // plain files: offset of the next unread byte
  size_t scan = 0;                   // scan state: bytes examined (see Fill)
  size_t chunk = 0;                  // bytes per read; 0 = 32 MB (gzip) / 128 MB (plain).  Set by the host test only.
  size_t file_bytes = 0, first_cut = 0;  // plain files: size; bytes of the first batch handed out (to size the record store)
  // One RawFile reads the files of a run one after the other: the buffer and its page lock stay from file to file
  bool Open(const std::string &path) {
    Close();
    have = 0; eof = false; scan = 0; nl = 0; fpos = 0; file_bytes = 0;
    unsigned char magic[2] = {0, 0};
    FILE *t = fopen(path.c_str(), "rb");
    if (!t) return false;
    const size_t got = fread(magic, 1, 2, t);
    fclose(t);
    if (got == 2 && magic[0] == 0x1f && magic[1] == 0x8b) { f = gzopen(path.c_str(), "rb"); if (f) gzbuffer(f, 1 << 20); return f != nullptr; }
    fd = open(path.c_str(), O_RDONLY);
    if (fd >= 0) { posix_fadvise(fd, 0, 0, POSIX_FADV_SEQUENTIAL); struct stat sb; if (fstat(fd, &sb) == 0) file_bytes = (size_t)sb.st_size; }
    return fd >= 0;
  }
  void Close() {
    if (f) gzclose(f);
    if (fd >= 0) close(fd);
    f = nullptr; fd = -1;
  }
  ~RawFile() {
    Close();
    if (pinned) cmx_host_unregister(buf.data());
  }
  void Reserve(size_t bytes, bool exact = false) {  // grow (rarely): the buffer is pinned once it has its working size
    if (buf.size() >= bytes) return;
    if (pinned) { cmx_host_unregister(buf.data()); pinned = false; }
    buf.Grow(exact ? bytes : bytes + bytes / 4, have);
    pinned = cmx_host_register(buf.data(), buf.size()) == 0;
  }
  // Size (and page-lock) the buffer for calls of max_records before the first one: bytes per record from the head of the file.
  // Run at start-up, beside the index upload, so that the mapping phase never allocates.
  void Prepare(uint32_t max_records) {
    if (f || fd < 0 || !file_bytes) return;
    std::vector<char> head(1u << 20);
    const ssize_t got = pread(fd, head.data(), head.size(), 0);
    if (got <= 0) return;
    const uint64_t lines = CountNewlines(head.data(), (size_t)got);
    if (lines < 8) return;
    const double per_record = (double)got / ((double)lines / 4.0);
    const size_t want = (size_t)(per_record * max_records * 1.1) + (128u << 20) + 4096;
    Reserve(std::min(want, file_bytes + 4096), true);
  }
  // bytes of up to max_records whole records now in the buffer (reading more as needed); *n = their number.
  // Newlines are counted in bulk (SSE2 compare + popcount, by the threads that read the data); only the stretch that holds
  // the last newline wanted is walked line by line.  State: nl = newlines in buf[0, scan).
  uint64_t nl = 0;
  static uint64_t CountNewlines(const char *p, size_t n) {
    uint64_t c = 0;
    size_t i = 0;
#if defined(__SSE2__)
    const __m128i v = _mm_set1_epi8('\n');
    for (; i + 64 <= n; i += 64) {
      const unsigned m0 = (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_loadu_si128((const __m128i *)(p + i)), v));
      const unsigned m1 = (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_loadu_si128((const __m128i *)(p + i + 16)), v));
      const unsigned m2 = (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_loadu_si128((const __m128i *)(p + i + 32)), v));
      const unsigned m3 = (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_loadu_si128((const __m128i *)(p + i + 48)), v));
      c += (uint64_t)__builtin_popcountll(((uint64_t)m0) | ((uint64_t)m1 << 16) | ((uint64_t)m2 << 32) | ((uint64_t)m3 << 48));
    }
#endif
    for (; i < n; ++i) c += p[i] == '\n';
    return c;
  }
  // advance the scan over buf[scan, scan + len) whose newline count is known; returns true once 4 * max_records are in
  bool Advance(size_t len, uint64_t count, uint64_t target) {
    if (nl + count < target) { nl += count; scan += len; return false; }
    while (nl < target) {  // the last newline wanted lies in this stretch
      const void *q = memchr(buf.data() + scan, '\n', have - scan);
      scan = (size_t)((const char *)q - buf.data()) + 1;
      ++nl;
    }
    return true;
  }
  uint64_t Fill(uint32_t max_records, uint32_t *n) {
    const uint64_t target = 4ull * max_records;
    if (max_records == 0) { *n = 0; return 0; }
    if (scan < have && nl < target) {  // what an earlier call left behind (less than one read chunk)
      const size_t len = have - scan;
      if (Advance(len, CountNewlines(buf.data() + scan, len), target)) { *n = max_records; return scan; }
    }
    for (;;) {
      if (nl >= target) { *n = max_records; return scan; }
      if (eof) {  // the file ended first: whole records only; up to three lines of an unfinished one stay behind
        const uint64_t whole = nl / 4;
        size_t e = have;
        for (uint64_t extra = nl - 4 * whole; extra > 0 && e > 0; --extra) {
          const void *q = memrchr(buf.data(), '\n', e - 1);  // the newline before the last line's own
          e = q ? (size_t)((const char *)q - buf.data()) + 1 : 0;
        }
        if (nl == 0) e = 0;
        *n = (uint32_t)whole;
        return whole ? e : 0;
      }
      size_t want = chunk ? chunk : (f ? (32u << 20) : (128u << 20));
      if (!f && !chunk && file_bytes)  // a plain file: never ask for more than is left (+ a few bytes, so that the end is seen as a short read)
        want = std::max<size_t>(64, std::min(want, file_bytes - std::min(file_bytes, fpos) + 8));
      Reserve(have + want + 1);
      if (f) {
        const long got = gzread(f, buf.data() + have, (unsigned)want);
        if (got <= 0) eof = true;
        else {
          have += (size_t)got;
          if (Advance((size_t)got, CountNewlines(buf.data() + scan, (size_t)got), target)) { *n = max_records; return scan; }
        }
      } else {  // plain file: eight threads pread() a slice each (one thread copies out of the page cache at 3-5 GB/s)
        const int nt = 8;
        const size_t slice = want / nt;
        size_t part[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint64_t cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        std::thread th[8];
        for (int t = 0; t < nt; ++t)
          th[t] = std::thread([&, t]() {
            size_t done = 0;
            char *dst = buf.data() + have + t * slice;
            while (done < slice) {
              const ssize_t r = pread(fd, dst + done, slice - done, (off_t)(fpos + t * slice + done));
              if (r <= 0) break;
              done += (size_t)r;
            }
            part[t] = done;
            cnt[t] = CountNewlines(dst, done);
          });
        for (int t = 0; t < nt; ++t) th[t].join();
        size_t got = 0;
        int used = 0;
        for (int t = 0; t < nt; ++t) { got += part[t]; ++used; if (part[t] < slice) break; }  // a short slice is the end of the file
        fpos += got;
        if (got == 0) eof = true;
        else {
          have += got;
          bool done = false;
          for (int t = 0; t < used && !done; ++t) done = Advance(part[t], cnt[t], target);
          if (done) { *n = max_records; return scan; }
        }
      }
      if (eof && have > 0 && buf[have - 1] != '\n') { buf[have++] = '\n'; ++nl; scan = have; }  // a last line without its newline
    }
  }
  void Consume(uint64_t bytes) {  // the remainder (less than one read chunk) is counted again by the next Fill
    if (!first_cut) first_cut = bytes;
    memmove(buf.data(), buf.data() + bytes, have - bytes);
    have -= bytes;
    scan = 0; nl = 0;
  }
};

static double g_t_fill = 0, g_t_ingest = 0;  // loader thread: reading + cutting, device-side parsing (summed over calls)

// --read-format: the ranges of read 1, read 2 and the barcode (whole reads without the option), and the refusal of reads
// the reference would cut in an undefined way (a read shorter than an explicit range end, nothing left after the cut)
struct ReadFormat {
  std::string text;
  cmx_read_range r[3];  // read 1, read 2, barcode
};
static void DieReadRange(const ReadFormat &rf, const std::string &detail) {
  Die("chromap-b200: --read-format " + rf.text + " does not fit the reads (" + detail + "); the reference's output is undefined for them");
}

// One batch through the device-side parser.  Returns false if a file is not plain 4-line FASTQ (the caller then uses the
// host reader); dies on real input errors, like LoadBatch.
static bool LoadBatchGpu(cmx_ctx *ctx, RawFile *f1, RawFile *f2, RawFile *fb, int parity, uint32_t max_pairs, Batch *b, bool keep_names, uint32_t bc_len,
                         const ReadFormat &rf) {
  b->Clear();
  uint32_t n1 = 0, n2 = 0, nb = 0;
  uint64_t c1 = 0, c2 = 0, cb = 0;  // the files are read (and inflated) side by side
  const double t_f0 = Now();
  std::thread t2, tb;
  if (f2) t2 = std::thread([&]() { c2 = f2->Fill(max_pairs, &n2); });
  if (fb) tb = std::thread([&]() { cb = fb->Fill(max_pairs, &nb); });
  c1 = f1->Fill(max_pairs, &n1);
  if (f2) t2.join();
  if (fb) tb.join();
  const double t_f1 = Now();
  g_t_fill += t_f1 - t_f0;
  if (n1 == 0 && n2 == 0 && nb == 0) {
    if (f1->have || (f2 && f2->have) || (fb && fb->have)) return false;  // trailing bytes that are no whole record: not 4-line FASTQ
    return true;
  }
  cmx_ingested g1{}, g2{}, gb{};
  std::vector<uint32_t> spans;
  if (keep_names) spans.resize(2 * (size_t)n1);
  auto ingest = [&](int which, RawFile *f, uint64_t bytes, int want_qual, uint32_t *name_spans, cmx_ingested *g) {
    const int rc = cmx_ingest_fastq_range(ctx, parity * 3 + which, f->buf.data(), bytes, want_qual, name_spans, &rf.r[which], g);
    if (rc == CMX_ERR_READ_RANGE) DieReadRange(rf, cmx_last_error(ctx));
    return rc == 0;
  };
  if (!ingest(0, f1, c1, 0, keep_names ? spans.data() : nullptr, &g1)) return false;
  if (f2 && !ingest(1, f2, c2, 0, nullptr, &g2)) return false;
  if (fb) {
    if (!ingest(2, fb, cb, 1, nullptr, &gb)) return false;
    if (nb && (gb.min_len != bc_len || gb.max_len != bc_len)) Die("ERROR: barcode lengths are not equal in the sample!");
  }
  // counted once every file is known to be 4-line FASTQ: a FASTA or multi-line mate goes to the host reader, which counts records
  if ((f2 && n2 != n1) || (fb && nb != n1)) Die("Numbers of reads and barcodes don't match!");
  if (keep_names) for (uint32_t i = 0; i < n1; ++i) b->names1.emplace_back(f1->buf.data() + spans[2 * i], spans[2 * i + 1]);
  g_t_ingest += Now() - t_f1;
  const double t_c0 = Now();
  f1->Consume(c1);
  if (f2) f2->Consume(c2);
  if (fb) fb->Consume(cb);
  g_t_fill += Now() - t_c0;
  b->n = n1; b->dev = true; b->max_len = std::max(g1.max_len, f2 ? g2.max_len : 0u);
  b->dev_in.n_pairs = n1; b->dev_in.seq1 = g1.seq; b->dev_in.off1 = g1.off; b->dev_in.on_device = 1;
  if (f2) { b->dev_in.seq2 = g2.seq; b->dev_in.off2 = g2.off; }
  if (fb) { b->dev_in.bc_seq = gb.seq; b->dev_in.bc_qual = gb.qual; b->dev_in.bc_len = bc_len; }
  return true;
}

// LoadPairedEndReadsWithBarcodes (chromap.cc:93-174, non-barcode): empty reads are skipped per file
// (sequence_batch.cc:28-31), the two files must run out together.
// utils.h:107-126
static uint64_t BarcodeSeed(const std::string &s) {
  uint64_t seed = 0;
  for (char c : s) {
    const int b = (c == 'A' || c == 'a') ? 0 : (c == 'C' || c == 'c') ? 1 : (c == 'G' || c == 'g') ? 2 : (c == 'T' || c == 't') ? 3 : 4;
    seed = b < 4 ? (seed << 2) | (uint64_t)b : seed << 2;
  }
  return seed;
}

// the cut of one read as loaded (sequence_batch.cc:35,51): reads the reference would cut in an undefined way are counted
static void CutRead(const cmx_read_range &r, std::string *s, std::string *q, uint32_t *n_short, uint32_t *n_empty) {
  const int64_t l = cmx_apply_read_range(&r, &(*s)[0], q->empty() ? nullptr : &(*q)[0], (uint32_t)s->size());
  if (l < 0) ++*n_short;
  else if (l == 0) ++*n_empty;
  s->resize(l < 0 ? 0 : (size_t)l);
  if (!q->empty()) q->resize(s->size());
}

static uint32_t LoadBatch(SeqReader &r1, SeqReader &r2, uint32_t max_pairs, Batch *b, bool keep_names, SeqReader *rb, uint32_t bc_len,
                          bool se, bool keep_sam, const ReadFormat &rf) {
  std::string n, s, q;
  uint32_t n_short = 0, n_empty = 0;
  b->Clear();
  while (b->n < max_pairs) {
    bool a = r1.Next(&n, &s, &q);
    while (a && s.empty()) a = r1.Next(&n, &s, &q);
    if (a) CutRead(rf.r[0], &s, &q, &n_short, &n_empty);
    if (a) { b->s1 += s; b->o1.push_back((uint32_t)b->s1.size()); if (keep_names) b->names1.push_back(n); if (keep_sam) { q.resize(s.size(), 'I'); b->q1 += q; } }
    bool c = a;  // single-end: no second file
    if (!se) {
      c = r2.Next(&n, &s, &q);
      while (c && s.empty()) c = r2.Next(&n, &s, &q);
      if (c) CutRead(rf.r[1], &s, &q, &n_short, &n_empty);
      if (c) { b->s2 += s; b->o2.push_back((uint32_t)b->s2.size()); if (keep_sam) { b->names2.push_back(n); q.resize(s.size(), 'I'); b->q2 += q; } }
    }
    bool d = c;
    if (rb) {
      d = rb->Next(&n, &s, &q);
      while (d && s.empty()) d = rb->Next(&n, &s, &q);
      if (d) CutRead(rf.r[2], &s, &q, &n_short, &n_empty);
      if (d && !n_short && !n_empty) {
        if (s.size() != bc_len) Die("ERROR: barcode lengths are not equal in the sample!");
        q.resize(bc_len, 'I');
        b->bc += s; b->bq += q;
      }
    }
    if (r1.Corrupted() || (!se && r2.Corrupted()) || (rb && rb->Corrupted())) Die("Didn't reach the end of sequence file, which might be corrupted!");  // sequence_batch.cc:46-55
    if (!a && !c && !d) break;
    if (a != c || c != d) Die("Numbers of reads and barcodes don't match!");
    ++b->n;
    b->max_len = std::max(b->max_len, b->o1[b->n] - b->o1[b->n - 1]);
    if (!se) b->max_len = std::max(b->max_len, b->o2[b->n] - b->o2[b->n - 1]);
  }
  if (n_short || n_empty)
    DieReadRange(rf, std::to_string(n_short) + " reads end before a range of the read format does, " + std::to_string(n_empty) + " reads are empty after the cut");
  return b->n;
}

// The command line (chromap_driver.cc:16-159), with the checks that need no device
struct Options {
  cmx_params p;
  std::string ref_path, index_path, r1_path, r2_path, out_path, bc_path, wl_path, tr_path;
  std::vector<std::string> r1_paths, r2_paths, bc_paths;  // -1 / -2 / -b expanded (ExpandReadPaths); set i = file i of each
  int k = 17, w = 7, bc_err = 1, out_nw = 0;
  bool allocate = false;                    // --allocate-multi-mappings (in-memory runs only, as the reference)
  int alloc_distance = 0, alloc_seed = 11;  // --multi-mapping-allocation-distance / -seed (mapping_parameters.h)
  double bc_prob = 0.9;
  bool build_index = false, skip_bc_check = false, host_reader = false, paf = false;
  bool cell_level_dedup = false;  // remove_pcr_duplicates_at_bulk_level == false (mapping_parameters.h:49; --preset atac clears it)
  bool cell_level_flag = false, bulk_level_flag = false;  // --remove-pcr-duplicates-at-cell-level / -at-bulk-level given
  ReadFormat rf;
  bool tagalign = false, sam = false, pairs = false, se = false, sc = false;  // output format (BED if none); -1 without -2; -b given
};
static Options ParseOptions(int argc, char **argv) {
  Options o;
  cmx_params &p = o.p;
  cmx_default_params(&p);
  std::string preset;
  for (int i = 1; i < argc; ++i)
    if (!strcmp(argv[i], "--preset") && i + 1 < argc) preset = argv[i + 1];
  if (cmx_apply_preset(&p, preset.c_str()) != 0) Die("Unrecognized preset parameters " + preset + "\n");
  if (preset == "atac") o.cell_level_dedup = true;  // chromap_driver.cc:254
  if (!preset.empty()) fprintf(stderr, "Preset parameters for %s are used.\n", preset.c_str());
  for (int i = 1; i + 1 < argc; ++i)
    if (!strcmp(argv[i], "--min-frag-length")) { const int l = atoi(argv[i + 1]); if (l <= 60) { o.k = 17; o.w = 7; } else if (l <= 80) { o.k = 19; o.w = 10; } else { o.k = 23; o.w = 11; } }
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto val = [&]() -> std::string { if (i + 1 >= argc) Die("Option " + a + " is missing an argument"); return argv[++i]; };
    if (a == "--preset") val();
    else if (a == "-i" || a == "--build-index") o.build_index = true;
    else if (a == "-h" || a == "--help") {
      printf("chromap-b200: chromap's paired-end BED path on H100 GPUs (subset of chromap options; see DESIGN.md)\n"
             "                      Reads of any length up to 832 bases map at full size: the mapping scratch grows to the longest read\n"
             "                      (--SAM: reads of up to 320 bases; a longer read stops the run before any output is written)\n"
             "  -1, -2, -b FILE     read 1, read 2 and cell barcode files: one path, a comma-separated list, or quoted glob patterns\n"
             "                      (e.g. -1 'L00*_R1.fq.gz'; each pattern's matches sorted, the lists in argument order).  File i of -1\n"
             "                      goes with file i of -2 and -b; each file starts new batches of 500,000 reads, as chromap\n"
             "  --read-format STR   parts of read 1, read 2 and the barcode to keep, as chromap: comma-separated r1|r2|bc:start:end[:+|-]\n"
             "                      (0-based, inclusive, end -1 = the last base; ranges of one file ascending, '-' reverse-complements)\n"
             "  --barcode-translate FILE  write barcoded BED fields and SAM CB:Z: tags through a TO,FROM (or TO<tab>FROM) table, plain or\n"
             "                      gzipped, as chromap (e.g. ATAC to gene-expression barcodes of 10x Multiome); bulk runs ignore it\n"
             "  --bc-error-threshold INT  max Hamming distance allowed to correct a barcode against the whitelist: 0, 1 or 2 [1]\n"
             "  --bc-probability-threshold FLT  min probability of the best correction among the candidates [0.9]\n"
             "  --allocate-multi-mappings  give each multi-mapped read (MAPQ < 4) one of its mappings, drawn with weights = the\n"
             "                      uni-mappings near it; reads with none nearby are dropped (in-memory BED / TagAlign runs; --low-mem\n"
             "                      and the presets ignore it)\n"
             "  --multi-mapping-allocation-distance INT  uni-mappings within this distance from any end of multi-mappings are used\n"
             "                      for allocation [0]\n"
             "  --multi-mapping-allocation-seed INT  seed for random number generator in multi-mapping allocation [11]\n"
             "  --remove-pcr-duplicates-at-bulk-level  with barcodes and --low-mem (the default there, as --preset chip): one record per\n"
             "                      position whatever its barcode, the barcode with the most duplicates, then the most abundant in the\n"
             "                      whitelist; needs --barcode-whitelist, not with --output-mappings-not-in-whitelist or --SAM\n"
             "  --remove-pcr-duplicates-at-cell-level  one record per position and barcode (as --preset atac); wins over the bulk level\n");
      exit(0);
    }
    else if (a == "-v" || a == "--version") { fprintf(stderr, "chromap-b200 0.1 (parity target: chromap 0.3.3-r521)\n"); exit(0); }
    else if (a == "-r" || a == "--ref") o.ref_path = val();
    else if (a == "-x" || a == "--index") o.index_path = val();
    else if (a == "-1" || a == "--read1") o.r1_path = val();
    else if (a == "-2" || a == "--read2") o.r2_path = val();
    else if (a == "-o" || a == "--output") o.out_path = val();
    else if (a == "-k" || a == "--kmer") o.k = atoi(val().c_str());
    else if (a == "-w" || a == "--window") o.w = atoi(val().c_str());
    else if (a == "--min-frag-length") val();  // applied before this loop: -k / -w always win over it (chromap_driver.cc:277-295)
    else if (a == "-e" || a == "--error-threshold") p.error_threshold = atoi(val().c_str());
    else if (a == "-s" || a == "--min-num-seeds") p.min_num_seeds = atoi(val().c_str());
    else if (a == "-f" || a == "--max-seed-frequencies") { const std::string v = val(); if (sscanf(v.c_str(), "%d,%d", &p.max_seed_freq0, &p.max_seed_freq1) != 2) Die("-f expects two comma separated integers"); }
    else if (a == "-l" || a == "--max-insert-size") p.max_insert_size = atoi(val().c_str());
    else if (a == "-q" || a == "--MAPQ-threshold") p.mapq_threshold = atoi(val().c_str());
    else if (a == "--min-read-length") p.min_read_length = atoi(val().c_str());
    else if (a == "--trim-adapters") p.trim_adapters = 1;
    else if (a == "--remove-pcr-duplicates") p.remove_pcr_duplicates = 1;
    else if (a == "--Tn5-shift") p.tn5_shift = 1;
    else if (a == "--low-mem") p.low_memory_mode = 1;
    else if (a == "--split-alignment") p.split_alignment = 1;
    else if (a == "--pairs") p.output_format = 5;
    else if (a == "-b" || a == "--barcode") o.bc_path = val();
    else if (a == "--barcode-whitelist") o.wl_path = val();
    else if (a == "--bc-error-threshold") o.bc_err = atoi(val().c_str());
    else if (a == "--bc-probability-threshold") o.bc_prob = atof(val().c_str());
    else if (a == "--output-mappings-not-in-whitelist") o.out_nw = 1;
    else if (a == "--barcode-translate") o.tr_path = val();
    else if (a == "--skip-barcode-check") o.skip_bc_check = true;
    else if (a == "--host-reader") o.host_reader = true;  // parse FASTQ on the host (multi-line records, FASTA reads)
    else if (a == "--read-format") o.rf.text = val();
    else if (a == "-n" || a == "--max-num-best-mappings") p.max_num_best_mappings = atoi(val().c_str());
    else if (a == "--drop-repetitive-reads") p.drop_repetitive_reads = atoi(val().c_str());
    else if (a == "--remove-pcr-duplicates-at-cell-level") o.cell_level_flag = true;   // chromap_driver.cc:395-400: the level only
    else if (a == "--remove-pcr-duplicates-at-bulk-level") o.bulk_level_flag = true;
    // options that cannot change BED / TagAlign / pairs output: host threads, the candidate cache (result-transparent), SAM scoring,
    // QC estimators; --BED, the default format
    else if (a == "-t" || a == "--num-threads" || a == "--cache-size" || a == "--cache-update-param" || a == "--frip-est-params" || a == "--k-for-minhash" || a == "-A" || a == "--match-score" ||
             a == "-B" || a == "--mismatch-penalty" || a == "-O" || a == "--gap-open-penalties" || a == "-E" || a == "--gap-extension-penalties") val();
    else if (a == "--BED" || a == "--debug-cache" || a == "--turn-off-num-uniq-cache-slots") {}
    else if (a == "--allocate-multi-mappings") o.allocate = true;
    else if (a == "--multi-mapping-allocation-distance") o.alloc_distance = atoi(val().c_str());
    else if (a == "--multi-mapping-allocation-seed") o.alloc_seed = atoi(val().c_str());
    else if (a == "--chr-order" || a == "--pairs-natural-chr-order" ||
             a == "-p" || a == "--matrix-output-prefix")
      Die("chromap-b200: option " + a + " changes the output in ways that are not on the GPU path; use the reference chromap for it");
    else if (a == "--TagAlign") p.output_format = 2;  // same records as BED, TagAlign / PairedTagAlign text (chromap_driver.cc:417-418)
    else if (a == "--SAM") p.output_format = 4;  // device: ksw spans, CIGARs, MAPQ, then order, NM / MD and the text (cmx_format_sam_gpu)
    else if (a == "--PAF") o.paf = true;  // BED-path records, PAF text and order on the host (cmx_format_paf)
    else if (a == "--summary")
      Die("chromap-b200: option " + a + " is not on the GPU path yet (BED and Hi-C pairs only); use the reference chromap for it");
    else Die("Unknown option " + a);
  }
  if (!o.bc_path.empty() && !o.wl_path.empty() && (o.bc_err < 0 || o.bc_err > 2))  // only a whitelist run corrects barcodes (chromap.h:897-909)
    Die("chromap-b200: --bc-error-threshold " + std::to_string(o.bc_err) + ": use 0, 1 or 2. A barcode is corrected by at most two substitutions; at " +
        "3 or more the reference lets that many Ns through but keeps the rest in the key as A, so the GPU path refuses it");
  const int rf_rc = cmx_parse_read_format(o.rf.text.c_str(), &o.rf.r[0], &o.rf.r[1], &o.rf.r[2]);  // chromap.cc:825-865
  if (rf_rc == CMX_ERR_INVALID) Die("Unknown read format: " + o.rf.text + "\n");
  if (rf_rc != CMX_OK)
    Die("chromap-b200: --read-format " + o.rf.text + ": the ranges of one file must ascend without overlapping, only the last may end at -1, and there may be up to " +
        std::to_string(CMX_MAX_READ_RANGES) + "; the reference runs such a format, but its in-place cut makes the result an artifact, so the GPU path refuses it");
  if (!(((p.output_format == 1 || p.output_format == 2 || p.output_format == 4) && !p.split_alignment) || (p.output_format == 5 && p.split_alignment)))
    Die("chromap-b200: supported outputs are BED / TagAlign (no split alignment) and Hi-C pairs (--split-alignment --pairs / --preset hic)");
  // chromap_driver.cc:395-400: the cell level wins whenever it is asked for, whatever the order; else the bulk level is asked for
  if (o.cell_level_flag) o.cell_level_dedup = true;
  else if (o.bulk_level_flag) o.cell_level_dedup = false;
  o.tagalign = p.output_format == 2; o.sam = p.output_format == 4; o.pairs = p.output_format == 5;
  o.se = o.r2_path.empty(); o.sc = !o.bc_path.empty();  // chromap_driver.cc:704-761: -1 alone = single-end
  return o;
}
// -i: the index built on the device, saved in the reference's file format (chromap_driver.cc:451-471)
static void BuildIndex(const Options &o, double t_start) {
  if (o.ref_path.empty() || o.out_path.empty()) Die("No reference specified!");
  fprintf(stderr, "Build index for the reference.\nKmer length: %d, window size: %d\nReference file: %s\nOutput file: %s\n", o.k, o.w, o.ref_path.c_str(), o.out_path.c_str());
  Reference ref;
  if (!ref.Load(o.ref_path)) Die("Cannot find sequence file " + o.ref_path);
  cmx_ctx *ctx = nullptr;
  const int rc = cmx_create(&ctx, 0, &o.p);
  if (rc) Die(rc == CMX_ERR_NO_DEVICE ? "chromap-b200: no CUDA device (there is no CPU fallback)" : "chromap-b200: cmx_create failed");
  if (cmx_upload_reference(ctx, (uint32_t)ref.names.size(), ref.offsets.data(), ref.concat.data())) Die(cmx_last_error(ctx));
  if (cmx_build_index(ctx, o.k, o.w)) Die(cmx_last_error(ctx));
  IndexFile ix;
  ix.k = o.k; ix.w = o.w;
  uint32_t n_occ = 0;
  if (cmx_download_index(ctx, &ix.n_buckets, &ix.size, nullptr, nullptr, nullptr, &n_occ, nullptr)) Die(cmx_last_error(ctx));
  ix.flags.resize(ix.n_buckets < 16 ? 1 : ix.n_buckets >> 4); ix.keys.resize(ix.n_buckets); ix.vals.resize(ix.n_buckets); ix.occ.resize(n_occ);
  if (cmx_download_index(ctx, &ix.n_buckets, &ix.size, ix.flags.data(), ix.keys.data(), ix.vals.data(), &n_occ, ix.occ.data())) Die(cmx_last_error(ctx));
  ix.n_occupied = ix.size;
  ix.upper_bound = (uint32_t)(ix.n_buckets * 0.77 + 0.5);
  if (!ix.Save(o.out_path)) Die("Cannot write index file " + o.out_path);
  fprintf(stderr, "Lookup table size: %u, # buckets: %u, occurrence table size: %u.\nBuilt and saved index in %.2fs.\n", ix.size, ix.n_buckets, n_occ, Now() - t_start);
  cmx_destroy(ctx);
}
// barcoded duplicates removed at bulk level: the low-memory merge's rule unless the cell level is asked for (mapping_writer.h:205-208)
static bool BulkLevelDedup(const Options &o) { return o.sc && o.p.remove_pcr_duplicates && o.p.low_memory_mode && !o.cell_level_dedup; }
// the checks of a mapping run that come after the -i branch, before any file is read or the device is touched
static void CheckMappingOptions(const Options &o) {
  if (o.ref_path.empty()) Die("No reference specified!");
  if (o.index_path.empty()) Die("No index specified!");
  if (o.r1_path.empty()) Die("No read file specified!");
  if (o.se && o.pairs) Die("chromap-b200: pairs output needs paired-end reads");
  if ((o.tagalign || o.paf) && o.sc) Die("chromap-b200: --TagAlign / --PAF with barcodes is not on the GPU path");
  if (o.paf && (o.sam || o.tagalign || o.pairs || o.p.trim_adapters)) Die("chromap-b200: --PAF goes with BED-path mapping without adapter trimming (trimmed read lengths are not returned yet)");
  if (o.pairs && o.p.remove_pcr_duplicates && !o.p.low_memory_mode)  // RemovePCRDuplicate keeps the LAST record of a run (mapping_processor.h:181-197): not on the GPU path for pairs
    Die("chromap-b200: duplicate removal of Hi-C pairs needs --low-mem (or --preset hic)");
  if (BulkLevelDedup(o)) {  // mapping_writer.h:205-208: only the low-memory merge has the bulk-level variant
    if (o.sam)  // IsSamePosition of SAM records compares the mate's rid with the line's own (sam_mapping.h)
      Die("chromap-b200: bulk-level duplicate removal of barcoded data is not on the GPU path (use --preset atac or --remove-pcr-duplicates-at-cell-level)");
    if (o.wl_path.empty())
      Die("chromap-b200: bulk-level duplicate removal of barcoded data ranks barcodes by their abundance in the whitelist; give --barcode-whitelist or "
          "--remove-pcr-duplicates-at-cell-level (without a whitelist the reference reads an empty table)");
    if (o.out_nw)
      Die("chromap-b200: bulk-level duplicate removal does not go with --output-mappings-not-in-whitelist: a barcode outside the whitelist has no "
          "abundance, and the reference reads past its table for it; use --remove-pcr-duplicates-at-cell-level");
  }
  if (o.out_path.empty()) Die("No output file specified!");
  if (o.allocate && !o.p.low_memory_mode) {  // low-memory runs accept the option and never allocate (chromap.h:605-613)
    if (o.alloc_distance < 0)
      Die("chromap-b200: --multi-mapping-allocation-distance " + std::to_string(o.alloc_distance) + ": use 0 or more; the reference casts a negative distance " +
          "to uint32, so its result is an accident of wrap-around, and the GPU path refuses it");
    if (o.sam || o.paf || o.pairs)
      Die("chromap-b200: --allocate-multi-mappings goes with BED / TagAlign output on the GPU path, not with --SAM, --PAF or --pairs");
  }
  if (o.allocate) fprintf(stderr, "Will allocate multi-mappings after mapping.\n");  // chromap_driver.cc:610-611
}
// The files of one -1 / -2 / -b argument (chromap_driver.cc:174-212): split at ',' as cxxopts splits a vector option (a trailing
// ',' adds nothing), each piece through glob(3) with ~ expanded; a pattern's matches come back sorted and are listed on stderr
static std::vector<std::string> ExpandPatterns(const std::string &arg) {
  std::vector<std::string> pieces, paths;
  size_t b = 0;
  for (size_t e; (e = arg.find(',', b)) != std::string::npos; b = e + 1) pieces.push_back(arg.substr(b, e - b));
  if (b < arg.size()) pieces.push_back(arg.substr(b));
  for (const std::string &pattern : pieces) {
    glob_t g;
    memset(&g, 0, sizeof(g));
    const int rc = glob(pattern.c_str(), GLOB_TILDE, nullptr, &g);
    if (rc == GLOB_NOMATCH) {  // the reference ends the run here too
      globfree(&g);
      Die(pattern.find_first_of("*?[") == std::string::npos ? "Cannot find sequence file " + pattern : "chromap-b200: no file matches " + pattern);
    }
    if (rc != 0) { globfree(&g); Die("glob() failed with return value " + std::to_string(rc) + " for " + pattern); }
    for (size_t i = 0; i < g.gl_pathc; ++i) {
      paths.push_back(g.gl_pathv[i]);
      fprintf(stderr, "%s\n", g.gl_pathv[i]);
    }
    globfree(&g);
  }
  return paths;
}
// -1, -2 and -b as lists of files, before any device work.  File i of -1 goes with file i of -2 and -b (chromap.h:801-812 loops
// over the -1 files): a shorter -2 or -b list would have the reference read past its end, so it is refused; the files of a
// longer one are never opened, as in the reference.
static void ExpandReadPaths(Options *o) {
  o->r1_paths = ExpandPatterns(o->r1_path);
  if (!o->se) o->r2_paths = ExpandPatterns(o->r2_path);
  if (o->sc) o->bc_paths = ExpandPatterns(o->bc_path);
  const size_t n = o->r1_paths.size();
  for (const auto &other : {std::make_pair("-2", &o->r2_paths), std::make_pair("-b", &o->bc_paths)}) {
    if (other.second->empty()) continue;  // not given
    const size_t m = other.second->size();
    if (m < n)
      Die(std::string("chromap-b200: ") + other.first + " lists " + std::to_string(m) + " file(s), -1 lists " + std::to_string(n) + ": file i of -1 goes with file i of " +
          other.first + ", so every -1 file needs one");
    if (m > n)
      fprintf(stderr, "WARNING: %s lists %zu file(s), -1 lists %zu: the last %zu file(s) of %s are not read.\n", other.first, m, n, m - n, other.first);
  }
}
// What a mapping run holds from start-up to exit: device context, reference, translation table, raw read files, record buffer
struct Session {
  cmx_ctx *ctx = nullptr;
  Reference ref;
  cmx_barcode_translation tr{};  // the writer loads the table in bulk runs too (mapping_writer.h:39-42), which then never use it
  RawFile g1, g2, gb;
  std::vector<cmx_pe_record> recs;
  std::vector<uint64_t> wl_keys;  // the whitelist and its abundances, for the host twin of bulk-level duplicate removal
  std::vector<uint32_t> wl_counts;
  bool gpu_reader = false, raw_ready = false, recs_pinned = false;  // raw_ready: g1 / g2 / gb hold the first call's reads
};
// Start-up, three things at once (the reference does them one after the other, chromap.h:684-730): the reference sequences
// are parsed by one thread, the index file is mapped and read ahead by the kernel, the CUDA context comes up on this thread
static void StartUp(const Options &o, double t_start, Session *s) {
  if (!o.tr_path.empty()) LoadBarcodeTranslation(o.tr_path, &s->tr);
  bool ref_ok = false;
  double t_ref_parsed = 0;
  std::thread ref_loader([&]() { ref_ok = s->ref.Load(o.ref_path); t_ref_parsed = Now(); });
  IndexMap ix;
  const bool ix_ok = ix.Open(o.index_path);
  const int rc = cmx_create(&s->ctx, 0, &o.p);
  if (!ix_ok) Die("Cannot load index file " + o.index_path);
  if (rc) Die(rc == CMX_ERR_NO_DEVICE ? "chromap-b200: no CUDA device (there is no CPU fallback)" : "chromap-b200: unsupported parameter combination");
  // the index arrays go to the device while the reference sequences are still being parsed — and while the first file set's
  // read files are opened, their page-locked buffers sized from the first records, and the first call's reads brought in
  s->gpu_reader = !o.host_reader && !o.sam && !o.paf;  // SAM / PAF keep names (SAM: bases and qualities too) of every read on the host
  const uint32_t first_call_pairs = (uint32_t)o.p.batch_size * 4u;
  std::thread raw_prep;
  if (s->gpu_reader) raw_prep = std::thread([&]() {
    if (!s->g1.Open(o.r1_paths[0]) || (!o.se && !s->g2.Open(o.r2_paths[0])) || (o.sc && !s->gb.Open(o.bc_paths[0]))) return;  // reported when the mapping opens them
    auto warm = [&](RawFile *f) { uint32_t n = 0; f->Prepare(first_call_pairs); f->Fill(first_call_pairs, &n); };
    std::thread a, b;
    if (!o.se) a = std::thread([&]() { warm(&s->g2); });
    if (o.sc) b = std::thread([&]() { warm(&s->gb); });
    warm(&s->g1);
    if (a.joinable()) a.join();
    if (b.joinable()) b.join();
    s->raw_ready = true;
  });
  const double t_ix = Now();
  if (cmx_upload_index(s->ctx, ix.k, ix.w, ix.n_buckets, ix.flags, ix.keys, ix.vals, ix.occ, ix.n_occ)) Die(cmx_last_error(s->ctx));
  fprintf(stderr, "Kmer size: %d, window size: %d.\nLookup table size: %u, occurrence table size: %u.\n", ix.k, ix.w, ix.size, ix.n_occ);
  ix.Close();
  const double t_ix_done = Now();
  ref_loader.join();
  if (!ref_ok) Die("Cannot find sequence file " + o.ref_path);
  fprintf(stderr, "Loaded all sequences successfully, number of sequences: %zu, number of bases: %zu.\n", s->ref.names.size(), s->ref.concat.size());
  const double t_ref = Now();
  if (cmx_upload_reference(s->ctx, (uint32_t)s->ref.names.size(), s->ref.offsets.data(), s->ref.concat.data())) Die(cmx_last_error(s->ctx));
  fprintf(stderr, "Start-up: context %.2fs, index to the device %.2fs, reference parsed (concurrently) after %.2fs, reference to the device %.2fs.\n", t_ix - t_start,
          t_ix_done - t_ix, t_ref_parsed - t_start, Now() - t_ref);
  if (raw_prep.joinable()) raw_prep.join();
  fprintf(stderr, "Reference and index resident on the device after %.2fs.\n", Now() - t_start);
}
// scATAC pre-pass (chromap.h:755-761): barcode length from the first record of the first barcode file, whitelist, abundance
// over the first >= 20 M whitelisted barcodes (chromap.cc:364-386, 388-548).  Returns the barcode length.
static uint32_t BarcodePrepass(const Options &o, Session &s) {
  if (o.pairs) Die("chromap-b200: barcodes with Hi-C pairs output are not on the GPU path");
  SeqReader rb0;
  OpenReads(&rb0, o.bc_paths[0]);
  std::string n, seq, q;
  uint32_t n_short = 0, n_empty = 0;
  auto cut = [&]() {  // every barcode is cut before its length or its key is looked at (chromap.cc:370, 494)
    CutRead(o.rf.r[2], &seq, &q, &n_short, &n_empty);
    if (n_short || n_empty) DieReadRange(o.rf, n_short ? "a barcode ends before a range of the read format does" : "a barcode is empty after the cut");
  };
  if (!rb0.Next(&n, &seq, &q)) Die("Empty barcode file");
  cut();
  const uint32_t bc_len = (uint32_t)seq.size();
  if (bc_len > 32) Die("ERROR: barcode length is greater than 32!");
  if (!o.wl_path.empty()) {
    std::unordered_map<uint64_t, uint32_t> wl;
    gzFile f = gzopen(o.wl_path.c_str(), "r");
    if (!f) Die("ERROR: barcode whitelist file does not exist or is truncated!");
    char buf[256];
    while (gzgets(f, buf, sizeof(buf)) != NULL) {
      size_t l = strlen(buf);
      if (l && buf[l - 1] == '\n') buf[--l] = 0;
      if (l != bc_len) Die(wl.empty() ? "ERROR: whitelist and input barcode lengths are not equal!" : "ERROR: barcode lengths are not equal in the whitelist!");
      wl.emplace(BarcodeSeed(std::string(buf, l)), 0u);
    }
    gzclose(f);
    fprintf(stderr, "Loaded %zu barcodes.\n", wl.size());
    // one reference batch at a time, file after file (the barcode file of each -1 file), batches restarting at every file; the
    // 5 % check compares the running total with the batch just counted; stop after the batch that reaches 20 M
    uint64_t num_sample = 0;
    for (size_t file = 0; file < o.r1_paths.size() && num_sample < 20000000ull; ++file) {
      SeqReader rb;
      OpenReads(&rb, o.bc_paths[file]);
      uint64_t in_batch = 0;
      bool more = true;
      while (more) {
        more = rb.Next(&n, &seq, &q);
        while (more && seq.empty()) more = rb.Next(&n, &seq, &q);
        if (more) {
          cut();
          if (seq.find('N') == std::string::npos) { auto it = wl.find(BarcodeSeed(seq)); if (it != wl.end()) { ++it->second; ++num_sample; } }
          ++in_batch;
        }
        if (in_batch == (uint64_t)o.p.batch_size || (!more && in_batch)) {
          if (!o.skip_bc_check && num_sample * 20 < in_batch) Die("Less than 5% barcodes can be found or corrected based on the barcode whitelist.");
          if (num_sample >= 20000000ull) break;
          in_batch = 0;
        }
      }
    }
    fprintf(stderr, "Compute barcode abundance using %llu.\n", (unsigned long long)num_sample);
    std::vector<uint64_t> &keys = s.wl_keys;
    std::vector<uint32_t> &counts = s.wl_counts;
    for (const auto &kv : wl) { keys.push_back(kv.first); counts.push_back(kv.second); }
    if (cmx_upload_barcode_whitelist(s.ctx, keys.data(), counts.data(), keys.size(), num_sample, bc_len, o.bc_err, o.bc_prob, o.out_nw)) Die(cmx_last_error(s.ctx));
  }
  if (!o.tr_path.empty() && cmx_upload_barcode_translation(s.ctx, &s.tr)) Die(cmx_last_error(s.ctx));
  return bc_len;
}
// What the writers need from the mapping calls, in read order
struct Mapped {
  bool sam, paf, se;
  std::vector<cmx_pe_record> all;           // BED-path records (cmx_pairs_record when pairs)
  std::vector<cmx_sam_record> sam_cores;    // SAM
  std::vector<uint64_t> bc;                 // barcode key of each record of `all`
  std::vector<std::string> names1, names2;  // read names, as the batches carry them (pairs: read 1; SAM / PAF: both)
  std::string s1, q1, s2, q2;               // SAM: bases and qualities of every read
  std::vector<uint64_t> off1{0}, off2{0};
  std::vector<uint16_t> len1, len2;         // PAF: read lengths
  uint64_t n_pairs = 0, n_mapped = 0, n_unique = 0, n_cand = 0, n_bc_in = 0, n_bc_cor = 0;
  void Append(const Batch &b, const cmx_records &out) {
    if (sam) {
      const cmx_sam_record *r = reinterpret_cast<const cmx_sam_record *>(out.records);
      sam_cores.insert(sam_cores.end(), r, r + out.n_records);
      for (uint32_t i = 0; i < b.n; ++i) { off1.push_back(off1.back() + (b.o1[i + 1] - b.o1[i])); if (!se) off2.push_back(off2.back() + (b.o2[i + 1] - b.o2[i])); }
      s1 += b.s1; q1 += b.q1; s2 += b.s2; q2 += b.q2;
    } else all.insert(all.end(), out.records, out.records + out.n_records);
    if (paf) for (uint32_t i = 0; i < b.n; ++i) { len1.push_back((uint16_t)(b.o1[i + 1] - b.o1[i])); if (!se) len2.push_back((uint16_t)(b.o2[i + 1] - b.o2[i])); }
    names1.insert(names1.end(), b.names1.begin(), b.names1.end());
    names2.insert(names2.end(), b.names2.begin(), b.names2.end());
    if (out.barcode_keys) bc.insert(bc.end(), out.barcode_keys, out.barcode_keys + out.n_records);
    n_pairs += b.n; n_mapped += out.n_mapped_pairs; n_unique += out.n_uniquely_mapped_pairs; n_cand += out.n_candidates;
    n_bc_in += out.n_barcodes_in_whitelist; n_bc_cor += out.n_barcodes_corrected;
  }
};
// The read files one set after the other (chromap.h:801-812): set i is file i of -1, -2 and -b.  A call never holds pairs of two
// sets, so every file starts a new reference batch at its first pair, as the reference's loader stops a batch at the end of a
// file (chromap.cc:93-116); the choice among equally good multi-mappings depends on a pair's place in its batch.  A set is
// parsed on the device when its files are plain 4-line FASTQ (decided on its first call), else by the host reader.
struct ReadSets {
  const Options &o;
  Session *s;
  uint32_t bc_len;
  size_t set = 0;                         // the set being read; o.r1_paths.size() once all are done
  bool on_device = false, first = true;   // first: the set's first call comes next
  SeqReader r1, r2, rb;
  ReadSets(const Options &o_, Session *s_, uint32_t bc_len_) : o(o_), s(s_), bc_len(bc_len_) {}
  // one call carries four reference batches (chromap.h:182: 500 000 pairs each) when the reads are parsed on the device: the
  // library runs them as overlapping lanes; batch boundaries stay where they are
  uint32_t CallPairs() const { return (uint32_t)o.p.batch_size * 4u; }
  void OpenHost() {
    if (o.sc) OpenReads(&rb, o.bc_paths[set]);
    OpenReads(&r1, o.r1_paths[set]);
    if (!o.se) OpenReads(&r2, o.r2_paths[set]);
  }
  // the first set: its raw files may already hold the first call's reads (StartUp)
  void Start() {
    set = 0; first = true; on_device = s->gpu_reader;
    if (!s->raw_ready) OpenSet();
  }
  void OpenSet() {
    if (set == o.r1_paths.size()) return;
    if (!on_device) { OpenHost(); return; }
    RawFile *files[3] = {&s->g1, o.se ? nullptr : &s->g2, o.sc ? &s->gb : nullptr};
    const std::string *paths[3] = {&o.r1_paths[set], o.se ? nullptr : &o.r2_paths[set], o.sc ? &o.bc_paths[set] : nullptr};
    for (int i = 0; i < 3; ++i)
      if (files[i]) { OpenReads(files[i], *paths[i]); files[i]->Prepare(CallPairs()); }  // (Prepare keeps a buffer that is large enough)
  }
  // The next call's reads into *b; b->n == 0 once every set is read.  A set that ends (or is empty) hands over to the next one.
  void Load(Batch *b, int parity) {
    for (; set < o.r1_paths.size(); ++set, first = true, on_device = s->gpu_reader, OpenSet()) {
      if (on_device && !LoadBatchGpu(s->ctx, &s->g1, o.se ? nullptr : &s->g2, o.sc ? &s->gb : nullptr, parity, CallPairs(), b, o.pairs, bc_len, o.rf)) {
        if (!first) Die(std::string("chromap-b200: the read files are not plain 4-line FASTQ (") + cmx_last_error(s->ctx) + "); rerun with --host-reader");
        fprintf(stderr, "Read files are not plain 4-line FASTQ (%s): using the host reader.\n", cmx_last_error(s->ctx));
        s->g1.Close(); s->g2.Close(); s->gb.Close();
        on_device = false;
        OpenHost();
      }
      if (!on_device) LoadBatch(r1, r2, (uint32_t)o.p.batch_size, b, o.pairs || o.sam || o.paf, o.sc ? &rb : nullptr, bc_len, o.se, o.sam || o.paf, o.rf);
      first = false;
      if (b->n) return;
    }
    b->Clear();
  }
};
// Bytes of the plain (not gzipped) files among paths: with the first call's bytes per pair, an estimate of the run's records
static size_t PlainFileBytes(const std::vector<std::string> &paths) {
  size_t total = 0;
  for (const std::string &p : paths) {
    FILE *t = fopen(p.c_str(), "rb");
    if (!t) continue;
    unsigned char magic[2] = {0, 0};
    struct stat sb;
    if (!(fread(magic, 1, 2, t) == 2 && magic[0] == 0x1f && magic[1] == 0x8b) && fstat(fileno(t), &sb) == 0) total += (size_t)sb.st_size;
    fclose(t);
  }
  return total;
}
// Reads longer than the context is sized for (cmx_params.max_read_length, 160 bases unless resized): before the call that
// holds them maps, the context grows to the call's longest read rounded up to a multiple of 32 bases (at most 832: the front
// end stages 64 reads per tile in shared memory, 227 KB on an H100; longer reads go to the overflow tiers).  Otherwise every
// such pair would take an overflow tier, sized for the few pairs a genome sends there.  SAM aligns reads of up to 320 bases: a longer read ends the run here, before any output file is written.
static void SizeForReads(const Options &o, cmx_ctx *ctx, uint32_t max_len, int32_t *L) {
  if ((int64_t)max_len <= *L) return;
  if (o.sam && max_len > 320)
    Die("chromap-b200: --SAM on the GPU path aligns reads of up to 320 bases, and a read of " + std::to_string(max_len) + " bases was found; no output file is written");
  const int32_t want = (int32_t)std::min<uint32_t>((max_len + 31) / 32 * 32, o.sam ? 320u : 832u);
  if (want <= *L) return;  // already at the largest size: the longer reads take the overflow tiers
  if (cmx_set_max_read_length(ctx, want)) Die(cmx_last_error(ctx));
  fprintf(stderr, "Reads of up to %u bases: mapping scratch resized for %d-base reads.\n", max_len, want);
  *L = want;
}
// Reference batches one library call maps at once.  Above 160 bases a call maps one batch at a time: a pair's tier-0
// scratch grows with the read length, and so does the share of pairs that reach the overflow tiers, which hold each such pair
// in megabytes (tier 2: about 3.5 MB).  On bench.py's 3 Gbp genome 0.48 % of 2x150 pairs reach tier 2 at 160 bases and
// 0.84 % of 2x250 pairs at 256 (DESIGN.md §9).  Batches stay whole, so the output does not change.
static uint32_t BatchesPerCall(int32_t L) { return L <= 160 ? 4u : 1u; }
// One loaded call through the library, BatchesPerCall(L) reference batches at a time; records and counters summed into *out.
static void MapCall(const Options &o, cmx_ctx *ctx, int32_t L, const cmx_batch &in, cmx_records *out, cmx_sam_record *sam_out) {
  const uint32_t step = BatchesPerCall(L) * (uint32_t)o.p.batch_size;
  cmx_records sum = *out;
  for (uint32_t p0 = 0; p0 < in.n_pairs; p0 += step) {
    cmx_batch part = in;
    part.n_pairs = std::min(step, in.n_pairs - p0);
    part.first_read_id += p0;
    part.off1 += p0;
    if (part.off2) part.off2 += p0;
    if (part.bc_seq) { part.bc_seq += (size_t)p0 * in.bc_len; part.bc_qual += (size_t)p0 * in.bc_len; }
    cmx_records r = *out;
    r.records = sam_out ? reinterpret_cast<cmx_pe_record *>(sam_out + sum.n_records) : out->records + sum.n_records;
    r.capacity = out->capacity - sum.n_records;
    if (out->barcode_keys) r.barcode_keys = out->barcode_keys + sum.n_records;
    if (cmx_map_batch_pe(ctx, &part, &r, nullptr)) Die(cmx_last_error(ctx));
    if (p0 == 0) { sum = r; sum.records = out->records; sum.capacity = out->capacity; sum.barcode_keys = out->barcode_keys; continue; }
    sum.n_records += r.n_records; sum.n_mapped_pairs += r.n_mapped_pairs; sum.n_uniquely_mapped_pairs += r.n_uniquely_mapped_pairs;
    sum.n_candidates += r.n_candidates; sum.n_overflow_pairs += r.n_overflow_pairs;
    sum.n_barcodes_in_whitelist += r.n_barcodes_in_whitelist; sum.n_barcodes_corrected += r.n_barcodes_corrected;
  }
  *out = sum;
}
// double-buffered batch loop: the loader thread prepares call c+1 while the GPU maps call c (chromap.h:871-877), opening the
// next file set when the current one ends, so a file switch overlaps the mapping of the set's last call.
static void MapReads(const Options &o, uint32_t bc_len, Session *s, Mapped *m) {
  cmx_ctx *ctx = s->ctx;
  ReadSets sets(o, s, bc_len);
  Batch cur, next;
  int parity = 0;
  sets.Start();
  if (s->gpu_reader) sets.Load(&cur, parity);
  const size_t r1_plain_bytes = s->gpu_reader ? PlainFileBytes(o.r1_paths) : 0;
  std::vector<cmx_pe_record> &recs = s->recs;
  const double t_map = Now();
  double t_calls = 0, t_collect = 0, t_wait = 0;
  int n_calls = 0;
  std::vector<cmx_sam_record> sam_recs;
  std::vector<uint64_t> bc_keys;
  int32_t read_len = o.p.max_read_length;  // what the context is sized for
  if (!s->gpu_reader) sets.Load(&cur, parity);
  while (cur.n > 0) {
    parity ^= 1;
    std::thread loader([&]() { sets.Load(&next, parity); });
    if (recs.size() < (size_t)cur.n * o.p.max_num_best_mappings) {  // the call's output buffer: page-locked, so the records come back at PCIe speed
      if (s->recs_pinned) { cmx_host_unregister(recs.data()); s->recs_pinned = false; }
      recs.resize((size_t)cur.n * o.p.max_num_best_mappings);
      s->recs_pinned = cmx_host_register(recs.data(), recs.size() * sizeof(cmx_pe_record)) == 0;
    }
    if (n_calls == 0 && cur.dev && r1_plain_bytes && s->g1.first_cut) {  // records of the whole run, from the first call's bytes per pair
      const double est = (double)r1_plain_bytes / (double)s->g1.first_cut * cur.n * 1.02 + 1024;
      if (est < 4e9) m->all.reserve((size_t)est);
    }
    cmx_batch in{};
    if (cur.dev) in = cur.dev_in;
    else {
      in.n_pairs = cur.n; in.seq1 = cur.s1.data(); in.off1 = cur.o1.data(); in.seq2 = o.se ? nullptr : cur.s2.data(); in.off2 = o.se ? nullptr : cur.o2.data();
      if (o.sc) { in.bc_seq = cur.bc.data(); in.bc_qual = cur.bq.data(); in.bc_len = bc_len; }
    }
    in.first_read_id = (uint32_t)m->n_pairs;  // the pairs of the earlier calls
    cmx_records out{};
    out.records = recs.data(); out.capacity = recs.size();
    if (o.sam) { sam_recs.resize(recs.size()); out.records = reinterpret_cast<cmx_pe_record *>(sam_recs.data()); }
    if (o.sc) { bc_keys.resize(recs.size()); out.barcode_keys = bc_keys.data(); }
    SizeForReads(o, ctx, cur.max_len, &read_len);
    const double t0 = Now();
    MapCall(o, ctx, read_len, in, &out, o.sam ? sam_recs.data() : nullptr);
    fprintf(stderr, o.se ? "Mapped %u reads in %.2fs.\n" : "Mapped %u read pairs in %.2fs.\n", cur.n, Now() - t0);
    t_calls += Now() - t0; ++n_calls;
    const double t_col0 = Now();
    m->Append(cur, out);
    const double t_j0 = Now();
    t_collect += t_j0 - t_col0;
    loader.join();
    t_wait += Now() - t_j0;
    std::swap(cur, next);
  }
  fprintf(stderr, "Mapped all reads in %.2fs.\n", Now() - t_map);
  fprintf(stderr, "Mapping phase: %d calls: mapping %.3fs, collecting records %.3fs, waiting for the loader %.3fs (loader: reading + cutting %.3fs, parsing on the device %.3fs, first batch included).\n",
          n_calls, t_calls, t_collect, t_wait, g_t_fill, g_t_ingest);
  fprintf(stderr, "Number of reads: %llu.\nNumber of mapped reads: %llu.\nNumber of uniquely mapped reads: %llu.\nNumber of candidates: %llu.\n",
          (unsigned long long)((o.se ? 1 : 2) * m->n_pairs), (unsigned long long)((o.se ? 1 : 2) * m->n_mapped), (unsigned long long)((o.se ? 1 : 2) * m->n_unique),
          (unsigned long long)m->n_cand);
}
// A text writer w(buf, cap) run for the length (buf == NULL), then into *text: the length, or the writer's negative status
template <class W> static int64_t Format(std::vector<char> *text, W w) {
  const int64_t bytes = w(nullptr, 0);
  if (bytes < 0) return bytes;
  text->resize((size_t)bytes + 1);
  return w(text->data(), bytes);
}
// The text written on the device; if either device call fails (records and text that do not fit beside the index), its host
// twin.  A barcode segment missing from the translation table ends the run instead, before any output is written.
template <class D, class H> static int64_t FormatOnDeviceElseHost(cmx_ctx *ctx, std::vector<char> *text, D dev, H host) {
  int64_t bytes = Format(text, dev);
  if (bytes == CMX_ERR_BARCODE_TRANSLATE) DieBarcodeNotTranslated(cmx_last_error(ctx));
  if (bytes >= 0) return bytes;
  bytes = Format(text, host);
  if (bytes == CMX_ERR_BARCODE_TRANSLATE) DieBarcodeNotTranslated("a barcode segment has no entry in the translation table");
  return bytes;
}
// --allocate-multi-mappings in an in-memory run: post-processing with the allocation on the device, its host twin if the device
// call fails for memory; the reference's log lines (mapping_processor.h:363,431-435, chromap.h:1348-1350).  A run without any
// multi-mapping ends here, before the output file is created (the reference aborts on an assertion).
static void Allocate(const Options &o, cmx_ctx *ctx, std::vector<cmx_pe_record> &all, uint64_t *bc, uint64_t *keep) {
  const double t0 = Now();
  cmx_allocation_stats st{};
  int rc = cmx_allocate_multi_mappings_gpu(ctx, all.data(), bc, all.size(), o.alloc_distance, o.alloc_seed, keep, &st);
  if (rc == CMX_ERR_CUDA) rc = cmx_allocate_multi_mappings(ctx, all.data(), bc, all.size(), o.alloc_distance, o.alloc_seed, keep, &st);
  if (rc) Die(std::string("chromap-b200: ") + cmx_last_error(ctx) + "; no output file is written");
  fprintf(stderr, "Got all %llu multi-mappings!\nAllocated %llu multi-mappings in %.2fs.\n# multi-mappings that have no uni-mapping overlaps: %llu.\n",
          (unsigned long long)st.n_multi, (unsigned long long)st.n_allocated, Now() - t0, (unsigned long long)st.n_without_overlap);
  fprintf(stderr, "After allocating multi-mappings, # uni-mappings: %llu, # multi-mappings: %llu, total: %llu.\n", (unsigned long long)st.n_uni_after,
          (unsigned long long)st.n_multi_after, (unsigned long long)(st.n_uni_after + st.n_multi_after));
}
// Post-processing (sort / dedup / filter on the device; the host routine if the records do not fit beside the index), text, file
static void WriteOutput(const Options &o, uint32_t bc_len, Session *s, Mapped *m, double t_start) {
  cmx_ctx *ctx = s->ctx;
  const Reference &ref = s->ref;
  const double t_pp = Now();
  std::vector<const char *> names, n1, n2;
  std::vector<uint32_t> lens;
  for (size_t i = 0; i < ref.names.size(); ++i) { names.push_back(ref.names[i].c_str()); lens.push_back((uint32_t)(ref.offsets[i + 1] - ref.offsets[i])); }
  for (const auto &x : m->names1) n1.push_back(x.c_str());
  for (const auto &x : m->names2) n2.push_back(x.c_str());
  std::vector<cmx_pe_record> &all = m->all;
  const bool allocate = o.allocate && !o.p.low_memory_mode;
  uint64_t keep = 0;
  std::vector<char> text;
  int64_t bytes = 0;
  if (o.sam) {  // bulk or barcoded (m->bc empty: bulk); the host twin without a table is exactly cmx_format_sam
    const cmx_read_set rs1{n1.data(), m->s1.data(), m->off1.data(), m->q1.data()}, rs2{n2.data(), m->s2.data(), m->off2.data(), m->q2.data()};
    const uint64_t *bc = o.sc ? m->bc.data() : nullptr;
    bytes = FormatOnDeviceElseHost(
        ctx, &text,
        [&](char *buf, int64_t cap) { return cmx_format_sam_gpu(ctx, names.data(), lens.data(), (uint32_t)names.size(), m->sam_cores.data(), bc, bc_len,
                                                                m->sam_cores.size(), &rs1, o.se ? nullptr : &rs2, 0, buf, cap); },
        [&](char *buf, int64_t cap) { return cmx_format_sam_bc(&o.p, names.data(), lens.data(), (uint32_t)names.size(), ref.concat.data(), ref.offsets.data(),
                                                               m->sam_cores.data(), bc, bc_len, m->sam_cores.size(), &rs1, o.se ? nullptr : &rs2, 0,
                                                               bc && !o.tr_path.empty() ? &s->tr : nullptr, buf, cap); });
    if (bytes < 0) Die("chromap-b200: the SAM writer failed (" + std::to_string(bytes) + ")");
    keep = (uint64_t)std::count(text.begin(), text.begin() + bytes, '\n') - names.size();  // less the @SQ header
    if (o.sc) fprintf(stderr, "Number of barcodes in whitelist: %llu.\nNumber of corrected barcodes: %llu.\n", (unsigned long long)m->n_bc_in, (unsigned long long)m->n_bc_cor);
  } else if (o.paf) {
    bytes = Format(&text, [&](char *buf, int64_t cap) { return cmx_format_paf(&o.p, names.data(), lens.data(), all.data(), all.size(), n1.data(), m->len1.data(),
                                                                              o.se ? nullptr : n2.data(), o.se ? nullptr : m->len2.data(), 0, buf, cap); });
    if (bytes < 0) Die("chromap-b200: cmx_format_paf failed");
    keep = (uint64_t)std::count(text.begin(), text.begin() + bytes, '\n');
    if (!o.se) keep /= 2;
  } else if (o.pairs) {
    cmx_pairs_record *pr = reinterpret_cast<cmx_pairs_record *>(all.data());
    if (cmx_postprocess_gpu(ctx, pr, nullptr, all.size(), &keep) && cmx_postprocess_pairs(ctx, pr, all.size(), &keep)) Die(cmx_last_error(ctx));
    bytes = FormatOnDeviceElseHost(
        ctx, &text, [&](char *buf, int64_t cap) { return cmx_format_pairs_gpu(ctx, names.data(), lens.data(), (uint32_t)names.size(), pr, keep, n1.data(), n1.size(), 0, buf, cap); },
        [&](char *buf, int64_t cap) { return cmx_format_pairs(names.data(), lens.data(), (uint32_t)names.size(), pr, keep, n1.data(), 0, buf, cap); });
  } else if (o.sc) {
    if (allocate) Allocate(o, ctx, all, m->bc.data(), &keep);
    else if (BulkLevelDedup(o)) {  // on the device, the host twin if the device call fails
      int rc = cmx_postprocess_bc_bulk_gpu(ctx, all.data(), m->bc.data(), all.size(), &keep);
      if (rc == CMX_ERR_CUDA) rc = cmx_postprocess_bc_bulk(&o.p, s->wl_keys.data(), s->wl_counts.data(), s->wl_keys.size(), all.data(), m->bc.data(), all.size(), &keep);
      if (rc) Die(std::string("chromap-b200: bulk-level duplicate removal failed: ") + cmx_last_error(ctx));
    } else if (cmx_postprocess_gpu(ctx, all.data(), m->bc.data(), all.size(), &keep) && cmx_postprocess_bc(ctx, all.data(), m->bc.data(), all.size(), &keep)) Die(cmx_last_error(ctx));
    bytes = FormatOnDeviceElseHost(  // the host twin without a table is exactly cmx_format_bed_bc
        ctx, &text, [&](char *buf, int64_t cap) { return cmx_format_bed_gpu(ctx, names.data(), all.data(), m->bc.data(), keep, bc_len, buf, cap); },
        [&](char *buf, int64_t cap) { return cmx_format_bed_bc_tr(names.data(), all.data(), m->bc.data(), keep, bc_len, o.tr_path.empty() ? nullptr : &s->tr, buf, cap); });
    fprintf(stderr, "Number of barcodes in whitelist: %llu.\nNumber of corrected barcodes: %llu.\n", (unsigned long long)m->n_bc_in, (unsigned long long)m->n_bc_cor);
  } else {
    if (allocate) Allocate(o, ctx, all, nullptr, &keep);
    else if (cmx_postprocess_gpu(ctx, all.data(), nullptr, all.size(), &keep) && cmx_postprocess(ctx, all.data(), all.size(), &keep)) Die(cmx_last_error(ctx));
    if (o.tagalign && !o.se)  // PairedTagAlign: two lines per pair (host formatter); single-end TagAlign is the BED text
      bytes = Format(&text, [&](char *buf, int64_t cap) { return cmx_format_tagalign(names.data(), all.data(), keep, buf, cap); });
    else
      bytes = FormatOnDeviceElseHost(
          ctx, &text, [&](char *buf, int64_t cap) { return cmx_format_bed_gpu(ctx, names.data(), all.data(), nullptr, keep, 0, buf, cap); },
          [&](char *buf, int64_t cap) { return cmx_format_bed(names.data(), all.data(), keep, buf, cap); });
  }
  FILE *fo = fopen(o.out_path.c_str(), "wb");
  if (!fo) Die("Cannot open output file " + o.out_path);
  fwrite(text.data(), 1, (size_t)bytes, fo);
  fclose(fo);
  fprintf(stderr, "Sorted, deduped and outputed mappings in %.2fs.\nNumber of output mappings (passed filters): %llu\nTotal time: %.2fs.\n", Now() - t_pp,
          (unsigned long long)keep, Now() - t_start);
}

int main(int argc, char **argv) {
  Options o = ParseOptions(argc, argv);
  const double t_start = Now();
  if (o.build_index) { BuildIndex(o, t_start); return 0; }
  CheckMappingOptions(o);
  ExpandReadPaths(&o);
  o.p.single_end = o.se ? 1 : 0;
  Session s;
  StartUp(o, t_start, &s);
  const uint32_t bc_len = o.sc ? BarcodePrepass(o, s) : 0;
  Mapped m{o.sam, o.paf, o.se};
  MapReads(o, bc_len, &s, &m);
  WriteOutput(o, bc_len, &s, &m, t_start);
  cmx_destroy(s.ctx);
  cmx_free_barcode_translation(&s.tr);
  return 0;
}
