"""The SAM text kernels of the CUDA path (chromap_b200/csrc/sam_text.cuh: line expansion, key words, run heads, survivor rule,
length pass with NM / MD / CB, write pass with one warp per line) run UNCHANGED on the host emulation (tests/cta_emu.h) in the
launch order of cmx_format_sam_gpu, with std::stable_sort in the place of CUB's radix passes (over the same key bits) and the
text written in two chunks; the text equals the host twin's (cmx_format_sam_bc / cmx_format_sam).  Inputs: the oracle's
barcoded cores and keys (tests/sam_bc_oracle.py), with and without a translation table and under both duplicate rules; bulk
synth_small cores (pe_chip, pe_q0d, se_n3, and atac-trimmed reads, whose CIGAR covers a prefix of the read); and a reference
with soft-masked and substituted bases inside the MD strings."""
import gzip
import os
import re
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests import emu
from tests import sam_bc_oracle as sbo
from tests.util import load_pairs, read_fasta, read_fastq_records

SMALL = os.path.join(sbo.GOLDEN, "synth_small")

MAIN = r'''
#include <string>
static std::vector<char> slurp(const std::string &p) { FILE *f = fopen(p.c_str(), "rb"); std::vector<char> v; char b[65536]; size_t n; if (!f) return v; while ((n = fread(b, 1, sizeof b, f)) > 0) v.insert(v.end(), b, b + n); fclose(f); return v; }
template <typename T> static std::vector<T> as(const std::vector<char> &v) { std::vector<T> o(v.size() / sizeof(T)); if (!o.empty()) memcpy(o.data(), v.data(), o.size() * sizeof(T)); return o; }
template <typename F> static void launch(size_t n, F body) { emu_grid_serial((int)((n + 255) / 256), 256, body); }
template <typename F> static void launch_warps(size_t n, F body) { emu_grid((int)((n + 255) / 256), 256, body); }   // (kernels with shuffles)
// CUB SortPairs(keys, idx, 0, bits): stable by the key's low `bits` bits
static void stable_by_key(std::vector<u64> &keys, std::vector<u32> &idx, int bits) {
  const u64 mask = bits >= 64 ? ~0ull : (1ull << bits) - 1;
  std::vector<u32> ord(keys.size());
  for (size_t i = 0; i < ord.size(); ++i) ord[i] = (u32)i;
  std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return (keys[a] & mask) < (keys[b] & mask); });
  std::vector<u32> ni(idx.size());
  for (size_t i = 0; i < ord.size(); ++i) ni[i] = idx[ord[i]];
  idx.swap(ni);
}
int main(int argc, char **argv) {
  // argv: dir; dir holds prm (i32: pe, bc_len, first_read_id, dedup, low_mem, mapq_threshold, has_bc, from_len), cores, bcs,
  // r{0,1}_{seq,qual,off,names,noff}, ref, ref_off, ref_names, ref_noff, tr_keys, tr_vals, tr_to
  const std::string d = std::string(argv[1]) + "/";
  const std::vector<int> prm = as<int>(slurp(d + "prm"));
  const int pe = prm[0], bc_len = prm[1], dedup = prm[3], low_mem = prm[4], mapq_threshold = prm[5], has_bc = prm[6], from_len = prm[7];
  const std::vector<OutSam> cores = as<OutSam>(slurp(d + "cores"));
  const std::vector<u64> bcs = as<u64>(slurp(d + "bcs"));
  std::vector<char> seq[2], qual[2], names[2];
  std::vector<u64> off[2], noff[2];
  SamText T{};
  T.cores = cores.data(); T.bcs = has_bc ? bcs.data() : nullptr; T.pe = pe; T.bc_len = bc_len; T.first_read_id = (u32)prm[2];
  for (int m = 0; m < (pe ? 2 : 1); ++m) {
    const std::string r = d + "r" + std::to_string(m) + "_";
    seq[m] = slurp(r + "seq"); qual[m] = slurp(r + "qual"); names[m] = slurp(r + "names");
    off[m] = as<u64>(slurp(r + "off")); noff[m] = as<u64>(slurp(r + "noff"));
    T.r[m] = SamReads{seq[m].data(), qual[m].empty() ? nullptr : qual[m].data(), off[m].data(), names[m].data(), noff[m].data()};
  }
  const std::vector<char> ref = slurp(d + "ref"), ref_names = slurp(d + "ref_names");
  const std::vector<u64> ref_off = as<u64>(slurp(d + "ref_off"));
  const std::vector<u32> ref_noff = as<u32>(slurp(d + "ref_noff"));
  T.ref = (const u8 *)ref.data(); T.ref_off = ref_off.data(); T.ref_names = ref_names.data(); T.ref_name_off = ref_noff.data();
  // the translation table as cmx_upload_barcode_translation lays it out
  std::vector<u64> tk = as<u64>(slurp(d + "tr_keys")), tv = as<u64>(slurp(d + "tr_vals"));
  std::vector<char> to = slurp(d + "tr_to");
  to.push_back(0);
  u64 ns = 64;
  while (ns < 2 * tk.size()) ns <<= 1;
  int lg = 0; while ((1ull << lg) < ns) ++lg;
  std::vector<ulonglong2> slots(ns, ulonglong2{CMX_EMPTY_KEY, CMX_EMPTY_KEY});
  launch(tk.size(), [&]() { tr_insert_kernel(tk.data(), tv.data(), tk.size(), slots.data(), ns - 1, 64 - lg); });
  unsigned long long n_missing = 0; unsigned first_missing = ~0u;
  BedTranslation Tr{};
  if (has_bc && from_len) { Tr.slots = slots.data(); Tr.mask = ns - 1; Tr.shift = 64 - lg; Tr.from_len = from_len; Tr.to = to.data(); Tr.n_missing = &n_missing; Tr.first_missing = &first_missing; }
  // cmx_format_sam_gpu's sequence
  const u64 n_lines = cores.size() * (pe ? 2 : 1);
  std::vector<u32> idx(n_lines);
  u64 max0 = 0;
  int err[2] = {0, 0};
  u32 max_ri = 0;
  launch_warps(n_lines, [&]() { sam_expand_kernel(T, n_lines, idx.data(), &max0, err); });
  launch_warps(n_lines, [&]() { sam_max_read_kernel(T, n_lines, &max_ri); });
  if (err[0]) { printf("overflow=%d\n", err[0]); return 0; }
  if ((u64)max_ri + 1 != off[0].size() - 1) { printf("bad read count %u\n", max_ri); return 1; }
  int bits0 = 1;
  while (bits0 < 64 && (max0 >> bits0)) ++bits0;
  std::vector<u64> keys(n_lines);
  for (int w = 3; w >= 0; --w) {
    if ((w == 1 && !has_bc) || (w == 2 && !pe)) continue;
    launch(n_lines, [&]() { sam_key_kernel(T, w, idx.data(), n_lines, keys.data()); });
    stable_by_key(keys, idx, w == 0 ? bits0 : w == 1 ? 2 * bc_len : w == 2 ? 32 : 41);
  }
  std::vector<u8> head(n_lines), keep(n_lines);
  std::vector<u32> res(n_lines), sel;
  launch(n_lines, [&]() { sam_head_kernel(T, dedup, idx.data(), n_lines, head.data()); });
  launch(n_lines, [&]() { sam_resolve_kernel(T, low_mem, mapq_threshold, idx.data(), head.data(), n_lines, res.data(), keep.data()); });
  for (u64 i = 0; i < n_lines; ++i) if (keep[i]) sel.push_back(res[i]);
  const u64 m = sel.size();
  std::vector<u32> len(m + 1, 0), nm(m, 0);
  launch(m, [&]() { sam_len_kernel(T, sel.data(), m, len.data(), nm.data(), err, Tr); });
  if (err[1]) { printf("long_cigar=%d\n", err[1]); return 0; }
  if (n_missing) { printf("missing=%llu first=%u\n", n_missing, first_missing); return 0; }
  std::vector<u64> toff(m + 1, 0);
  for (u64 i = 0; i < m; ++i) toff[i + 1] = toff[i] + len[i];
  std::string text((size_t)toff[m], '?');
  const u64 CH = m / 2 + 1;   // two chunks, the second written at a base that is not 0
  for (u64 c0 = 0; c0 < m; c0 += CH) {
    const u64 k = std::min(CH, m - c0);
    launch(k * 32, [&]() { sam_write_kernel(T, sel.data() + c0, k, toff.data() + c0, toff[c0], nm.data() + c0, &text[toff[c0]], Tr); });
  }
  FILE *f = fopen((d + "text").c_str(), "wb"); fwrite(text.data(), 1, text.size(), f); fclose(f);
  printf("lines=%llu bytes=%llu\n", (unsigned long long)m, (unsigned long long)text.size());
  return 0;
}
'''


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    return emu.build(tmp_path_factory.mktemp("samtext"), emu.PIPELINE + ["postprocess.cuh", "sam_text.cuh"], MAIN)


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def _emu(exe, d, p, names, seqs, cores, bcs, bc_len, reads1, reads2, translation=None):
    """Runs the kernels on the emulator: (status fields, text without the @SQ header)."""
    pe = reads2 is not None
    np.array([int(pe), bc_len, 0, p.remove_pcr_duplicates, p.low_memory_mode, p.mapq_threshold, int(bcs is not None),
              translation.from_len if translation is not None else 0], dtype=np.int32).tofile(str(d / "prm"))
    np.ascontiguousarray(cores).tofile(str(d / "cores"))
    _u64(bcs if bcs is not None else []).tofile(str(d / "bcs"))
    n_reads = int(cores["read_id"].max()) + 1
    for m, r in enumerate([reads1] + ([reads2] if pe else [])):
        nm, sq, ql = (x[:n_reads] for x in r)
        (d / ("r%d_seq" % m)).write_bytes(b"".join(sq)); (d / ("r%d_qual" % m)).write_bytes(b"".join(ql))
        (d / ("r%d_names" % m)).write_bytes(b"".join(nm))
        _u64(np.concatenate([[0], np.cumsum([len(x) for x in sq])])).tofile(str(d / ("r%d_off" % m)))
        _u64(np.concatenate([[0], np.cumsum([len(x) for x in nm])])).tofile(str(d / ("r%d_noff" % m)))
    (d / "ref").write_bytes(b"".join(bytes(s) for s in seqs))
    _u64(np.concatenate([[0], np.cumsum([len(s) for s in seqs])[:-1]])).tofile(str(d / "ref_off"))
    (d / "ref_names").write_bytes("".join(names).encode())
    np.concatenate([[0], np.cumsum([len(s) for s in names])]).astype(np.uint32).tofile(str(d / "ref_noff"))
    t = translation if translation is not None else cb.BarcodeTranslation([0], [b""], 1)
    to_off = np.concatenate([[0], np.cumsum([len(x) for x in t.to])]).astype(np.uint64)
    (to_off[:-1] << np.uint64(16) | _u64([len(x) for x in t.to])).tofile(str(d / "tr_vals"))
    t.keys.tofile(str(d / "tr_keys")); (d / "tr_to").write_bytes(b"".join(t.to))
    r = subprocess.run([str(exe), str(d)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    f = dict(kv.split("=") for kv in r.stdout.split() if "=" in kv)
    return f, ((d / "text").read_bytes() if "lines" in f else None)


def _strip_header(text, n_seq):
    at = 0
    for _ in range(n_seq):
        at = text.index(b"\n", at) + 1
    return text[at:]


def _check(exe, d, p, names, seqs, cores, bcs, bc_len, reads1, reads2, translation=None):
    want = cb.format_sam_bc(p, names, seqs, cores, bcs, bc_len, reads1, reads2, translation=translation)
    f, text = _emu(exe, d, p, names, seqs, cores, bcs, bc_len, reads1, reads2, translation)
    assert text is not None, f
    assert int(f["lines"]) > 500
    assert text == _strip_header(want, len(names))
    return want


def _sc_inputs(name):
    ref, index, r1, r2 = sbo.setup()
    keys, ok, bc_len = sbo.barcode_gate(name)
    se = sbo.RUNS[name][2]
    cores, ck = sbo.cores_and_keys(sbo.params(name), index, ref, r1, None if se else r2, keys, ok)
    names, seqs = read_fasta(os.path.join(sbo.SC, "ref.fa.gz"))
    reads = lambda recs: ([r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs])
    return names, seqs, cores.view(cb.SAM_RECORD), ck, bc_len, reads(r1), None if se else reads(r2)


def _cb_params(name, **kw):
    preset, over, se, _, _, _, _, _ = sbo.RUNS[name]
    return cb.make_params(preset, output_format=4, single_end=int(se), **dict(over, **kw))


@pytest.mark.parametrize("name,kw", [("pe_atac", {}), ("se_atac", {}), ("pe_q0dedup", {}), ("pe_q0dedup", dict(low_memory_mode=1)),
                                     ("se_q0dedup", dict(low_memory_mode=1)), ("pe_n3q0", {}), ("pe_half8", {}), ("pe_rc16", {})])
def test_barcoded_cores(emu_exe, tmp_path, name, kw):
    names, seqs, cores, ck, bc_len, reads1, reads2 = _sc_inputs(name)
    tr_path = sbo.RUNS[name][7]
    t = cb.parse_barcode_translation(gzip.open(tr_path).read()) if tr_path else None
    want = _check(emu_exe, tmp_path, _cb_params(name, **kw), names, seqs, cores, ck, bc_len, reads1, reads2, t)
    if not kw:
        assert want == gzip.open(os.path.join(sbo.OUT, name + ".sam.gz")).read()


def test_missing_translation_segment(emu_exe, tmp_path):
    names, seqs, cores, ck, bc_len, reads1, reads2 = _sc_inputs("pe_atac")
    t = cb.parse_barcode_translation(gzip.open(os.path.join(sbo.TR, "missing_rc16.txt.gz")).read())
    f, text = _emu(emu_exe, tmp_path, _cb_params("pe_atac"), names, seqs, cores, ck, bc_len, reads1, reads2, t)
    assert text is None and int(f["missing"]) > 0
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_sam_bc(_cb_params("pe_atac"), names, seqs, cores, ck, bc_len, reads1, reads2, translation=t)


def _small_inputs(preset, paired, **kw):
    names, seqs = read_fasta(os.path.join(SMALL, "ref.fa.gz"))
    ref = orc.Reference(os.path.join(SMALL, "ref.fa.gz"))
    idx = orc.Index(ref=ref, k=17, w=7)
    s1, o1, s2, o2 = load_pairs(SMALL)
    cores = orc.map_sam_cores(orc.make_params(preset, **kw), idx, ref, s1, o1, s2 if paired else None, o2 if paired else None).view(cb.SAM_RECORD)
    split = lambda r: ([a for a, _, _ in r], [b for _, b, _ in r], [c for _, _, c in r])
    r1 = split(read_fastq_records(os.path.join(SMALL, "read1.fq.gz")))
    r2 = split(read_fastq_records(os.path.join(SMALL, "read2.fq.gz"))) if paired else None
    p = cb.make_params(preset, max_read_length=64, output_format=4, single_end=0 if paired else 1, **kw)
    return p, names, seqs, cores, r1, r2


@pytest.mark.parametrize("case,preset,kw,paired", [("pe_chip", "chip", {}, True), ("pe_q0d", "", dict(mapq_threshold=0, remove_pcr_duplicates=1), True),
                                                   ("se_n3", "", dict(max_num_best_mappings=3, mapq_threshold=0), False),
                                                   ("pe_atac_q0", "atac", dict(mapq_threshold=0), True)])
def test_bulk_cores(emu_exe, tmp_path, case, preset, kw, paired):
    p, names, seqs, cores, r1, r2 = _small_inputs(preset, paired, **kw)
    if preset == "atac":  # adapter trimming: some CIGARs cover only a prefix of their read
        rl = lambda c, m: sum(int(x) >> 4 for x in c["cigar"][m][:c["n_cigar"][m]] if int(x) & 0xF != 2)
        assert sum(rl(c, 0) < len(r1[1][c["read_id"]]) for c in cores) > 10
    want = _check(emu_exe, tmp_path, p, names, seqs, cores, None, 0, r1, r2)
    if case != "pe_atac_q0":
        assert want == gzip.open(os.path.join(SMALL, case + ".sam.gz")).read()


def test_soft_masked_reference_inside_md(emu_exe, tmp_path):
    """Every 5th reference base in lower case and every 17th replaced by another lower-case base: MD prints them as stored."""
    p, names, seqs, cores, r1, r2 = _small_inputs("", True, mapq_threshold=0)
    masked = []
    for s in seqs:
        s = s.copy()
        s[::5] = np.char.lower(s[::5].view("S1")).view(np.uint8)
        sub = s[::17]
        s[::17] = np.frombuffer(b"cgta", dtype=np.uint8)[np.searchsorted(np.frombuffer(b"ACGT", dtype=np.uint8), np.char.upper(sub.view("S1")).view(np.uint8)) % 4]
        masked.append(s)
    want = _check(emu_exe, tmp_path, p, names, masked, cores, None, 0, r1, r2)
    assert len(re.findall(rb"MD:Z:[0-9ACGT^]*[acgt]", want)) > 100


BYTES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "synth_bytes")


@pytest.mark.parametrize("case,reads,paired", [("pe_q0.sam", "pe100", True), ("se_q0.sam", "pe100", False), ("pe250_q0.sam", "pe250", True)])
def test_cores_on_raw_bytes(emu_exe, tmp_path, case, reads, paired):
    """Reads with lower case, 'n', '.', IUPAC codes and high bytes on a soft-masked reference with IUPAC codes and bytes 0x80-0xFF
    (tests/golden/synth_bytes): the minus-strand SEQ turns every byte that is no base into 'N', NM / MD compare the read's raw
    bytes against the reference folded to upper case and print the reference bytes as stored.  Device text == host twin ==
    the reference binary's output."""
    names, seqs = read_fasta(os.path.join(BYTES, "ref.fa.gz"))
    ref = orc.Reference(os.path.join(BYTES, "ref.fa.gz"))
    s1, o1, s2, o2 = load_pairs(BYTES, reads + "_1.fq.gz", reads + "_2.fq.gz")
    cores = orc.map_sam_cores(orc.make_params("", mapq_threshold=0), orc.Index(ref=ref, k=17, w=7), ref, s1, o1,
                              s2 if paired else None, o2 if paired else None).view(cb.SAM_RECORD)
    split = lambda r: ([a for a, _, _ in r], [b for _, b, _ in r], [c for _, _, c in r])
    r1 = split(read_fastq_records(os.path.join(BYTES, reads + "_1.fq.gz")))
    r2 = split(read_fastq_records(os.path.join(BYTES, reads + "_2.fq.gz"))) if paired else None
    p = cb.make_params("", max_read_length=256, output_format=4, single_end=int(not paired), mapq_threshold=0)
    want = _check(emu_exe, tmp_path, p, names, seqs, cores, None, 0, r1, r2)
    assert want == gzip.open(os.path.join(BYTES, case + ".gz")).read()
    # the bytes reached the text: MD strings that name lower-case or high reference bytes
    assert len(re.findall(rb"MD:Z:[^\t\n]*[acgt\x80-\xff]", want)) > 100
