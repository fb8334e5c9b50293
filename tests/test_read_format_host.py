"""--read-format without a GPU: the parser (cmx_parse_read_format) against a table of accepted and refused strings, the host
cut (cmx_apply_read_range) against a literal restatement of SequenceEffectiveRange::Replace (sequence_effective_range.h:
80-118), the device cut (ingest.cuh: ingest_cut_len_kernel, ingest_cut_pack_kernel) run unchanged on the host emulation in
cmx_ingest_fastq_range's sequence against the host cut, and the CLI's handling of the option before it needs a device."""
import ctypes as C
import os
import random
import subprocess

import pytest

import chromap_b200 as cb
from tests import emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
WHOLE = [(0, -1)]
ERR_INVALID, ERR_READ_RANGE = -3, -7

# format -> (r1, r2, bc), each (ranges, reverse)
ACCEPTED = {
    "": ((WHOLE, 0), (WHOLE, 0), (WHOLE, 0)),
    "bc:0:15": ((WHOLE, 0), (WHOLE, 0), ([(0, 15)], 0)),
    "bc:8:23": ((WHOLE, 0), (WHOLE, 0), ([(8, 23)], 0)),
    "bc:0:15:-": ((WHOLE, 0), (WHOLE, 0), ([(0, 15)], 1)),
    "bc:0:15:+": ((WHOLE, 0), (WHOLE, 0), ([(0, 15)], 0)),
    "bc:0:7,bc:12:19": ((WHOLE, 0), (WHOLE, 0), ([(0, 7), (12, 19)], 0)),
    "bc:0:15,r1:16:-1": (([(16, -1)], 0), (WHOLE, 0), ([(0, 15)], 0)),
    "r1:0:39,r2:5:-1": (([(0, 39)], 0), ([(5, -1)], 0), (WHOLE, 0)),
    "r2:0:-1:-": ((WHOLE, 0), (WHOLE, 1), (WHOLE, 0)),
    "r1:0:-1:-": ((WHOLE, 1), (WHOLE, 0), (WHOLE, 0)),
    "bc:0:7:-,bc:12:19": ((WHOLE, 0), (WHOLE, 0), ([(0, 7), (12, 19)], 1)),     # the strand is per file: the last one given wins
    "bc:0:7:-,bc:12:19:+": ((WHOLE, 0), (WHOLE, 0), ([(0, 7), (12, 19)], 0)),
    "r1:3:3": (([(3, 3)], 0), (WHOLE, 0), (WHOLE, 0)),
    "r1:007:9": (([(7, 9)], 0), (WHOLE, 0), (WHOLE, 0)),
    "bc:0:3,r1:4:9,bc:8:11,r2:1:2:-,bc:20:-1": (([(4, 9)], 0), ([(1, 2)], 1), ([(0, 3), (8, 11), (20, -1)], 0)),
    ",".join("r1:%d:%d" % (2 * k, 2 * k) for k in range(8)): (([(2 * k, 2 * k) for k in range(8)], 0), (WHOLE, 0), (WHOLE, 0)),
}
# outside the grammar: "Unknown read format" (several of them the reference's hand parser accepts, with accidental meanings)
MALFORMED = ["r1x:0:5", "r3:0:5", "rr:0:5", "R1:0:5", "b:0:5", "r1:0", "r1", "r1:0:5:", "r1:0:5:x", "r1:0:5:++", "r1:0:5:-:", "r1:0:5:-:+",
             "r1:-1:5", "r1:5:3", "r1:a:5", "r1:0:b", "r1:+0:5", "r1:0:-2", "r1: 0:5", "r1 :0:5", "r1:0:1234567890", "r1:0:5,",
             ",r1:0:5", "r1:0:5,,r2:0:5", "r1::5", "r1:0:"]
# in the grammar, but the reference's in-place cut makes the result an artifact: refused
REFUSED = ["r1:5:9,r1:0:3", "r1:0:5,r1:5:9", "r1:0:-1,r1:5:9", "bc:0:-1,bc:20:-1", "bc:4:7,bc:0:1:-",
           ",".join("r1:%d:%d" % (2 * k, 2 * k) for k in range(9))]


def _parse(fmt):
    L = cb.load_library()
    r = [cb.ReadRange() for _ in range(3)]
    return L.cmx_parse_read_format(fmt.encode(), *[C.byref(x) for x in r]), r


@pytest.mark.parametrize("fmt", sorted(ACCEPTED))
def test_parser_accepts(fmt):
    rc, r = _parse(fmt)
    assert rc == 0
    assert [(x.ranges(), x.reverse) for x in r] == [(list(a), b) for a, b in ACCEPTED[fmt]]
    assert [(x.ranges(), x.reverse) for x in cb.parse_read_format(fmt)] == [(list(a), b) for a, b in ACCEPTED[fmt]]


@pytest.mark.parametrize("fmt", MALFORMED)
def test_parser_refuses_malformed(fmt):
    assert _parse(fmt)[0] == ERR_INVALID
    with pytest.raises(cb.CmxError, match="Unknown read format"):
        cb.parse_read_format(fmt)


@pytest.mark.parametrize("fmt", REFUSED)
def test_parser_refuses_ranges_the_reference_cuts_as_an_artifact(fmt):
    assert _parse(fmt)[0] == ERR_READ_RANGE


# ---- the host cut against Replace, restated line by line (utils.h:87-100 for the complement)
def _char_to_uint8(c):
    return {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3, ord("a"): 0, ord("c"): 1, ord("g"): 2, ord("t"): 3}.get(c, 4)


def _replace(starts, ends, strand, s, need_complement):
    s = bytearray(s) + b"\0"
    n = len(s) - 1
    if strand == "+" and starts[0] == 0 and ends[0] == -1:
        return bytes(s[:n])
    i = 0
    for k in range(len(starts)):
        start, end = starts[k], ends[k]
        if end == -1:
            end = n - 1
        j = start
        while j <= end:
            s[i] = s[j]
            i += 1
            j += 1
    s[i] = 0
    n = i
    if strand == "-":
        if need_complement:
            for i in range(n):
                s[i] = b"ACGTNNNN"[3 ^ _char_to_uint8(s[i])]
        i, j = 0, n - 1
        while i < j:
            s[i], s[j] = s[j], s[i]
            i += 1
            j -= 1
    return bytes(s[:n])


def _random_format(rng, which, max_start):
    """A random format in the grammar with ascending, disjoint ranges; returns (text, starts, ends, strand)."""
    n = rng.randint(1, 8) if rng.random() < 0.2 else rng.randint(1, 3)
    starts, ends, pos = [], [], 0
    for k in range(n):
        a = pos + rng.randint(0, max_start // n)
        if k + 1 == n and rng.random() < 0.4:
            e = -1
        else:
            e = a + rng.randint(0, 12)
        starts.append(a)
        ends.append(e)
        pos = e + 1
    strand = rng.choice("+-")
    fields = ["%s:%d:%d" % (which, a, e) for a, e in zip(starts, ends)]
    if strand == "-" or rng.random() < 0.3:
        k = rng.randrange(n)
        fields[k] += ":" + strand
    return ",".join(fields), starts, ends, strand


def test_host_cut_equals_replace():
    L = cb.load_library()
    rng = random.Random(29)
    alphabet = b"ACGTNacgtn" * 4 + bytes(range(1, 256))
    counts = {"cut": 0, "short": 0, "empty": 0, "rev": 0}
    for it in range(6000):
        which = rng.choice(["r1", "r2", "bc"])
        fmt, starts, ends, strand = _random_format(rng, which, 40)
        r = cb.parse_read_format(fmt)[{"r1": 0, "r2": 1, "bc": 2}[which]]
        assert r.ranges() == list(zip(starts, ends)) and r.reverse == (strand == "-"), fmt
        n = rng.randint(1, 70)
        seq = bytes(rng.choice(alphabet) for _ in range(n))
        qual = bytes(rng.randint(33, 126) for _ in range(n))
        s, q = C.create_string_buffer(seq, n), C.create_string_buffer(qual, n)
        with_qual = it % 3 != 0
        got = L.cmx_apply_read_range(C.byref(r), s, q if with_qual else None, n)
        if any(e != -1 and e >= n for e in ends):   # Replace would read past the read: undefined, refused
            assert got == ERR_READ_RANGE, (fmt, n)
            counts["short"] += 1
            continue
        want_s = _replace(starts, ends, strand, seq, True)
        want_q = _replace(starts, ends, strand, qual, False)
        assert got == len(want_s), (fmt, seq, got)
        if got == 0:
            counts["empty"] += 1
            continue
        assert s.raw[:got] == want_s, (fmt, seq)
        if with_qual:
            assert q.raw[:got] == want_q, (fmt, qual)
        assert s.raw[got:] == seq[got:]   # nothing past the cut is touched
        counts["cut"] += 1
        counts["rev"] += strand == "-"
    assert counts["cut"] > 2000 and counts["short"] > 300 and counts["empty"] > 20 and counts["rev"] > 1000, counts


# ---- the device cut on the host emulation
MAIN = r'''
#include <random>
static const char *kAlphabet = "ACGTNacgtnACGTACGTRYK.*";
static cmx_read_range random_range(std::mt19937 &g) {
  cmx_read_range r{};
  r.n = g() % 5 == 0 ? 1 + g() % CMX_MAX_READ_RANGES : 1 + g() % 3;
  int pos = 0;
  for (u32 k = 0; k < r.n; ++k) {
    r.start[k] = pos + (int)(g() % (60 / r.n + 1));
    r.end[k] = k + 1 == r.n && g() % 5 < 2 ? -1 : r.start[k] + (int)(g() % 25);
    pos = r.end[k] + 1;
  }
  r.reverse = g() % 2;
  return r;
}
int main() {
  std::mt19937 g(107);
  long bad = 0, n_records = 0, n_short = 0, n_empty = 0, n_cut = 0, n_rev = 0;
  for (int it = 0; it < 160; ++it) {
    const bool crlf = it % 4 == 1, want_qual = it % 3 != 2;
    const cmx_read_range range = random_range(g);
    CutRanges cr{range.n, {}, {}, range.reverse};
    for (u32 k = 0; k < range.n; ++k) { cr.start[k] = range.start[k]; cr.end[k] = range.end[k]; }
    const int n = 1 + (int)(g() % 300);
    std::string text;
    std::vector<std::string> seqs, quals;
    auto eol = [&]() { if (crlf) text.push_back('\r'); text.push_back('\n'); };
    for (int r = 0; r < n; ++r) {
      const int L = 1 + (int)(g() % 120);
      std::string s, q;
      for (int i = 0; i < L; ++i) { s.push_back(kAlphabet[g() % strlen(kAlphabet)]); q.push_back((char)(33 + g() % 60)); }
      text += "@read" + std::to_string(r); eol();
      text += s; eol();
      text += "+"; eol();
      text += q; eol();
      seqs.push_back(s); quals.push_back(q);
    }
    // cmx_ingest_fastq_range's sequence: newline flags, compaction, records, cut lengths, scan, cut pack
    const u32 nb = (u32)text.size();
    std::vector<u8> flag(nb + 1);
    emu_grid_serial((int)((nb + 255) / 256), 256, [&]() { newline_flag_kernel(text.data(), nb, flag.data()); });
    std::vector<u32> nl;
    for (u32 i = 0; i < nb; ++i) if (flag[i]) nl.push_back(i);
    std::vector<u32> seq_start(n + 1), qual_start(n + 1), len(n + 1, 0), off(n + 1, 0);
    IngestStats st{0, 0, 0, 0, 0xFFFFFFFFu, 0};
    CutStats cs{0, 0, 0xFFFFFFFFu, 0};
    emu_grid_serial((n + 255) / 256, 256, [&]() { ingest_record_kernel(text.data(), nl.data(), (u32)n, seq_start.data(), qual_start.data(), len.data(), nullptr, &st); });
    emu_grid_serial((n + 255) / 256, 256, [&]() { ingest_cut_len_kernel(len.data(), (u32)n, cr, &cs); });
    for (int i = 0; i < n; ++i) off[i + 1] = off[i] + len[i];
    std::string seq(text.size() + 64, '?'), qual(text.size() + 64, '?');
    emu_grid_serial((int)(((u64)n * 32 + 255) / 256), 256, [&]() {
      ingest_cut_pack_kernel(text.data(), seq_start.data(), qual_start.data(), off.data(), nl.data(), (u32)n, cr, &seq[0], want_qual ? &qual[0] : nullptr);
    });
    // the host cut of every record
    u32 want_short = 0, want_empty = 0, mn = 0xFFFFFFFFu, mx = 0;
    bool ok = st.bad_header == 0 && st.bad_plus == 0 && st.empty_reads == 0 && st.qual_mismatch == 0;
    for (int r = 0; r < n && ok; ++r) {
      std::string s = seqs[r], q = quals[r];
      const int64_t c = cmx_apply_read_range(&range, &s[0], &q[0], (u32)s.size());
      const u32 l = off[r + 1] - off[r], want_l = c < 0 ? 0u : (u32)c;
      if (c == CMX_ERR_READ_RANGE) ++want_short;
      else if (c == 0) ++want_empty;
      else if (c < 0) ok = false;
      mn = std::min(mn, want_l); mx = std::max(mx, want_l);
      ok = ok && l == want_l && memcmp(seq.data() + off[r], s.data(), l) == 0 && (!want_qual || memcmp(qual.data() + off[r], q.data(), l) == 0);
      if (c > 0) { ++n_cut; n_rev += range.reverse; }
      ++n_records;
    }
    ok = ok && cs.out_of_range == want_short && cs.empty == want_empty && cs.min_len == mn && cs.max_len == mx;
    ok = ok && seq.compare(off[n], 64, std::string(64, '?')) == 0 && (!want_qual || qual.compare(off[n], 64, std::string(64, '?')) == 0);  // nothing written past the cut
    n_short += want_short; n_empty += want_empty;
    if (!ok) { if (bad < 6) printf("CUT it=%d crlf=%d qual=%d n=%d ranges=%u rev=%d short %u/%u empty %u/%u\n", it, crlf, want_qual, n, range.n, range.reverse, cs.out_of_range, want_short, cs.empty, want_empty); ++bad; }
  }
  printf("records=%ld cut=%ld reversed=%ld short=%ld empty=%ld bad=%ld\n", n_records, n_cut, n_rev, n_short, n_empty, bad);
  return bad != 0;
}
'''


def test_device_cut_kernels_equal_the_host_cut(tmp_path):
    lib = cb.lib_path()
    cb.load_library()
    out = emu.run(tmp_path, ["device_common.cuh", "ingest.cuh"], MAIN, timeout=1200,
                  flags=["-include", os.path.join(ROOT, "include", "chromap_b200.h")], libs=[lib, "-Wl,-rpath," + os.path.dirname(lib)])
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["cut"]) > 5000 and int(f["reversed"]) > 2000 and int(f["short"]) > 1000 and int(f["empty"]) > 50, out.stdout


# ---- the CLI, before it needs a device
def _cli(*args):
    if not os.path.exists(CLI):
        import __graft_entry__
        __graft_entry__.build()
    d = os.path.join(ROOT, "tests", "golden", "ref_test")
    return subprocess.run([CLI, "-x", os.path.join(d, "ref.index"), "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "read1.fq"),
                           "-2", os.path.join(d, "read2.fq"), "-o", "/tmp/never.bed"] + list(args), capture_output=True, text=True)


def test_cli_read_format_parses_and_reaches_the_device_gate():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present: the gate is not reached")
    for fmt in ("bc:0:15", "r1:0:39,r2:5:-1", "r2:0:-1:-", ""):
        r = _cli("--read-format", fmt)
        assert r.returncode != 0 and "no CPU fallback" in r.stderr, (fmt, r.stderr)


def test_cli_read_format_refusals_before_the_device():
    r = _cli("--read-format", "r1x:0:5")
    assert r.returncode != 0 and "Unknown read format: r1x:0:5" in r.stderr, r.stderr
    r = _cli("--read-format", "bc:8:15,bc:0:7")
    assert r.returncode != 0 and "the reference runs such a format" in r.stderr and "GPU path refuses it" in r.stderr, r.stderr
    r = _cli("--read-format")
    assert r.returncode != 0 and "missing an argument" in r.stderr, r.stderr
