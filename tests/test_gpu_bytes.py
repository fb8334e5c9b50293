"""GPU parity on reads and a reference beyond upper-case ACGTN (tests/golden/synth_bytes, see tests/test_oracle_bytes.py): a
soft-masked reference with IUPAC codes and bytes 0x80-0xFF, reads with lower case, 'n', '.', IUPAC codes and high bytes.
- cmx_build_index on the golden reference and on a reference holding every byte 0x01-0xFF has the content of `chromap -i`;
- every case through the library, from an uploaded and from a device-built index: records and SAM cores field by field against
  the oracle, BED / TagAlign / SAM / pairs text byte for byte against the reference binary's golden; the 2x250 cases in a
  context created at 160 bases and grown by cmx_set_max_read_length;
- every golden through chromap-b200, with the device reader and with --host-reader.
Run with `-m gpu` on an H100."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.test_gpu_parity import _read_names, assert_same_records
from tests.test_oracle_bytes import CASES, CUT_COMPLEMENT, REF_BIN, all_bytes_reference, index_content
from tests.util import pack, read_fasta, read_fastq, read_fastq_records

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
READ_LEN = {"pe100": 100, "hic150": 150, "pe250": 250}


@pytest.fixture(scope="module")
def byte_set(golden_dir):
    d = os.path.join(golden_dir, "synth_bytes")
    names, seqs = read_fasta(os.path.join(d, "ref.fa.gz"))
    oref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    reads = {}
    for r in READ_LEN:
        a, b = read_fastq(os.path.join(d, r + "_1.fq.gz")), read_fastq(os.path.join(d, r + "_2.fq.gz"))
        reads[r] = (*pack(a), *pack(b))
    # rf_rev's --read-format r1:0:-1:-,r2:0:-1:- cuts each mate to its reverse complement ("ACGTNNNN"[3 ^ CharToUint8(c)])
    a, b = read_fastq(os.path.join(d, "pe100_1.fq.gz")), read_fastq(os.path.join(d, "pe100_2.fq.gz"))
    cut = lambda r: CUT_COMPLEMENT[np.frombuffer(r, dtype=np.uint8)[::-1]].tobytes()
    reads["rf_rev"] = (*pack([cut(r) for r in a]), *pack([cut(r) for r in b]))
    return dict(d=d, names=names, seqs=seqs, oref=oref, oidx=orc.Index(ref=oref, k=17, w=7), reads=reads)


def _index_equals_reference_binary(m, ref_fa, tmp_path):
    subprocess.check_call([REF_BIN, "-i", "-r", ref_fa, "-o", str(tmp_path / "ref.index")], stderr=subprocess.DEVNULL)
    theirs = index_content(orc.Index(str(tmp_path / "ref.index")).arrays())
    m.build_index(17, 7)
    ours = index_content(m.download_index())
    assert theirs[0] == ours[0] and np.array_equal(theirs[1], ours[1]) and theirs[2] == ours[2]
    return len(ours[2])


@pytest.mark.parametrize("which", ["golden", "every_byte"])
def test_device_built_index_has_the_content_of_the_reference_binarys_index(byte_set, which, tmp_path):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    if which == "golden":
        fa = str(tmp_path / "ref.fa")
        open(fa, "wb").write(gzip.open(os.path.join(byte_set["d"], "ref.fa.gz")).read())
        names, seqs = byte_set["names"], byte_set["seqs"]
    else:
        text, seqs = all_bytes_reference()
        fa = str(tmp_path / "ref.fa")
        open(fa, "wb").write(text)
        names = ["s%d" % i for i in range(len(seqs))]
    m = cb.Mapper(cb.make_params("", max_read_length=64))
    m.upload_reference(seqs, names)
    assert _index_equals_reference_binary(m, fa, tmp_path) > 40000


def _mapper(s, on_device, preset, max_read_length, grow_to=None, **kw):
    m = cb.Mapper(cb.make_params(preset, max_read_length=max_read_length, **kw))
    m.upload_reference(s["seqs"], s["names"])
    if on_device:
        m.build_index(17, 7)
    else:
        a = s["oidx"].arrays()
        m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    if grow_to:
        m.set_max_read_length(grow_to)
    return m


def _context(reads):
    """(max_read_length the context is created at, the length it is grown to or None): reads of up to 160 bases in a context of
    at most the default 160, longer ones in a default context grown to 256"""
    L = READ_LEN.get(reads, 100)
    return (160, 256) if L > 160 else (min(160, L + 28), None)


LIB_CASES = sorted(c for c in CASES if not c.endswith(".paf"))


@pytest.mark.parametrize("on_device", [False, True], ids=["uploaded_index", "device_built_index"])
@pytest.mark.parametrize("case", LIB_CASES)
def test_records_and_text_on_raw_bytes_equal_oracle_and_golden(byte_set, case, on_device):
    s = byte_set
    preset, kw, reads, paired, _ = CASES[case]
    if case == "rf_rev.bed":
        reads = "rf_rev"
    mrl, grow = _context(reads)
    s1, o1, s2, o2 = s["reads"][reads]
    want = gzip.open(os.path.join(s["d"], case + ".gz")).read()
    op = orc.make_params(preset, **kw, single_end=int(not paired))
    if case.endswith(".sam"):
        m = _mapper(s, on_device, preset, mrl, grow, output_format=4, single_end=int(not paired), **kw)
        if not paired:
            s2 = o2 = None
        recs, stats = m.map_batch(s1, o1, s2, o2)
        cores = orc.map_sam_cores(op, s["oidx"], s["oref"], s1, o1, s2, o2)
        assert len(recs) == len(cores) > 500 and stats["n_overflow_pairs"] == 0
        for f in ("read_id", "rid", "mapq", "is_unique", "secondary", "overflow"):
            assert np.array_equal(recs[f], cores[f]), f
        for q in range(2 if paired else 1):
            for f in ("pos", "end", "strand", "n_cigar"):
                assert np.array_equal(recs[f][:, q], cores[f][:, q]), (f, q)
            for i in range(len(recs)):
                n = recs["n_cigar"][i, q]
                assert np.array_equal(recs["cigar"][i, q, :n], cores["cigar"][i, q, :n]), (i, q)
        split = lambda r: ([a for a, _, _ in r], [b for _, b, _ in r], [c for _, _, c in r])
        r1 = split(read_fastq_records(os.path.join(s["d"], reads + "_1.fq.gz")))
        r2 = split(read_fastq_records(os.path.join(s["d"], reads + "_2.fq.gz"))) if paired else None
        assert cb.format_sam(m.params, s["names"], s["seqs"], recs, r1, r2) == want
        assert m.format_sam_gpu(recs, r1, r2) == want
        return
    m = _mapper(s, on_device, preset, mrl, grow, single_end=int(not paired), **kw)
    if paired:
        recs, stats = m.map_batch(s1, o1, s2, o2)
        orecs, _ = orc.map_pairs(op, s["oidx"], s["oref"], s1, o1, s2, o2)
    else:
        recs, stats = m.map_batch(s1, o1, None, None)
        orecs = orc.map_reads_se(op, s["oidx"], s["oref"], s1, o1)
    assert len(recs) == len(orecs) > 500 and stats["n_overflow_pairs"] == 0
    assert_same_records(recs, orecs)
    if case.endswith(".pairs"):
        rn = _read_names(os.path.join(s["d"], reads + "_1.fq.gz"))
        lens = [len(x) for x in s["seqs"]]
        assert m.format_pairs(m.postprocess_pairs(recs), rn, lens) == want
        assert m.format_pairs_gpu(m.postprocess_gpu(recs), rn, lens) == want
    elif case.endswith(".tagalign"):
        assert m.format_tagalign(m.postprocess(recs)) == want
    else:
        assert m.format_bed(m.postprocess(recs)) == want
        assert m.format_bed_gpu(m.postprocess_gpu(recs)) == want


@pytest.fixture(scope="module")
def cli_index(byte_set, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ix") / "bytes.index")
    subprocess.check_call([CLI, "-i", "-r", os.path.join(byte_set["d"], "ref.fa.gz"), "-o", out], stderr=subprocess.DEVNULL)
    return out


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_cli_on_raw_bytes_equals_reference_binary_output(byte_set, cli_index, case, reader, tmp_path):
    d = byte_set["d"]
    _, _, reads, paired, opts = CASES[case]
    out = str(tmp_path / case)
    args = [CLI, "-x", cli_index, "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, reads + "_1.fq.gz")]
    args += ["-2", os.path.join(d, reads + "_2.fq.gz")] if paired else []
    r = subprocess.run(args + opts + ["-o", out] + (["--host-reader"] if reader == "host" else []), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if reader == "device":
        assert "using the host reader" not in r.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(d, case + ".gz")).read()
