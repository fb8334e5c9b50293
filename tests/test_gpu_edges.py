"""GPU parity at the ends of reference sequences and on references of many short sequences, through the C ABI: the synth_edges
inputs (tests/golden/synth_edges: a 60 kbp sequence and 50 short ones, 70% of the fragments within 40 bp of a sequence's ends)
field by field against the CPU oracle and byte for byte against the reference binary's outputs; and a reference of 70,000 short
sequences (rid > 2^16 in the post-processing sort keys, the pairs keys and the text kernels' name offsets) against the oracle.
Run with `-m gpu` on an H100."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.test_gpu_parity import _read_names, assert_same_records
from tests.test_oracle_edges import EDGE_CASES, assert_reaches_the_edges
from tests.util import load_pairs, pack, read_fasta, read_fastq_records

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")


@pytest.fixture(scope="module")
def edges(golden_dir):
    d = os.path.join(golden_dir, "synth_edges")
    names, seqs = read_fasta(os.path.join(d, "ref.fa.gz"))
    oref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    return dict(d=d, names=names, seqs=seqs, oref=oref, oidx=orc.Index(ref=oref, k=17, w=7), pairs=load_pairs(d),
                hic_pairs=load_pairs(d, "hic_read1.fq.gz", "hic_read2.fq.gz"))


def _mapper(edges, on_device, preset, **kw):
    m = cb.Mapper(cb.make_params(preset, **kw))
    m.upload_reference(edges["seqs"], edges["names"])
    if on_device:
        m.build_index(17, 7)
    else:
        a = edges["oidx"].arrays()
        m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    return m


@pytest.mark.parametrize("on_device", [False, True], ids=["uploaded_index", "device_built_index"])
@pytest.mark.parametrize("case", sorted(c for c in EDGE_CASES if c.endswith(".bed")))
def test_bed_records_at_sequence_ends_equal_oracle_and_golden(edges, case, on_device):
    preset, kw, paired, _ = EDGE_CASES[case]
    m = _mapper(edges, on_device, preset, max_read_length=64, single_end=int(not paired), **kw)
    op = orc.make_params(preset, **kw)
    s1, o1, s2, o2 = edges["pairs"]
    if paired:
        recs, stats = m.map_batch(s1, o1, s2, o2)
        orecs, _ = orc.map_pairs(op, edges["oidx"], edges["oref"], s1, o1, s2, o2)
    else:
        recs, stats = m.map_batch(s1, o1, None, None)
        orecs = orc.map_reads_se(op, edges["oidx"], edges["oref"], s1, o1)
    assert len(recs) == len(orecs) > 1000 and stats["n_overflow_pairs"] == 0
    assert_same_records(recs, orecs)
    want = gzip.open(os.path.join(edges["d"], case + ".gz")).read()
    assert m.format_bed(m.postprocess(recs)) == want
    assert m.format_bed_gpu(m.postprocess_gpu(recs)) == want
    assert_reaches_the_edges(case, want, dict(zip(edges["names"], map(len, edges["seqs"]))))


@pytest.mark.parametrize("on_device", [False, True], ids=["uploaded_index", "device_built_index"])
@pytest.mark.parametrize("paired", [True, False], ids=["pe", "se"])
def test_sam_cores_at_sequence_ends_equal_oracle(edges, paired, on_device):
    m = _mapper(edges, on_device, "", max_read_length=64, output_format=4, mapq_threshold=0, single_end=int(not paired))
    s1, o1, s2, o2 = edges["pairs"]
    if not paired:
        s2 = o2 = None
    recs, stats = m.map_batch(s1, o1, s2, o2)
    cores = orc.map_sam_cores(orc.make_params("", mapq_threshold=0, single_end=int(not paired)), edges["oidx"], edges["oref"], s1, o1, s2, o2)
    assert len(recs) == len(cores) > 1000 and stats["n_overflow_pairs"] == 0
    for f in ("read_id", "rid", "mapq", "is_unique", "secondary", "overflow"):
        assert np.array_equal(recs[f], cores[f]), f
    for q in range(2 if paired else 1):
        for f in ("pos", "end", "strand", "n_cigar"):
            bad = np.nonzero(recs[f][:, q] != cores[f][:, q])[0]
            assert len(bad) == 0, (f, q, bad[:5], recs[f][bad[:5], q], cores[f][bad[:5], q])
        for i in range(len(recs)):
            n = recs["n_cigar"][i, q]
            assert np.array_equal(recs["cigar"][i, q, :n], cores["cigar"][i, q, :n]), (i, q)
    split = lambda r: ([a for a, _, _ in r], [b for _, b, _ in r], [c for _, _, c in r])
    r1 = split(read_fastq_records(os.path.join(edges["d"], "read1.fq.gz")))
    r2 = split(read_fastq_records(os.path.join(edges["d"], "read2.fq.gz"))) if paired else None
    text = cb.format_sam(m.params, edges["names"], edges["seqs"], recs, r1, r2)
    case = ("pe" if paired else "se") + "_q0.sam"
    assert text == gzip.open(os.path.join(edges["d"], case + ".gz")).read()
    assert_reaches_the_edges(case, text, dict(zip(edges["names"], map(len, edges["seqs"]))))


@pytest.mark.parametrize("on_device", [False, True], ids=["uploaded_index", "device_built_index"])
def test_hic_pairs_at_sequence_ends_equal_oracle_and_golden(edges, on_device):
    m = _mapper(edges, on_device, "hic", max_read_length=160, mapq_threshold=0)
    s1, o1, s2, o2 = edges["hic_pairs"]
    recs, stats = m.map_batch(s1, o1, s2, o2)
    orecs, _ = orc.map_pairs(orc.make_params("hic", mapq_threshold=0), edges["oidx"], edges["oref"], s1, o1, s2, o2)
    assert len(recs) == len(orecs) > 500 and stats["n_overflow_pairs"] == 0
    assert_same_records(recs, orecs)
    rn = _read_names(os.path.join(edges["d"], "hic_read1.fq.gz"))
    lens = [len(s) for s in edges["seqs"]]
    text = m.format_pairs(m.postprocess_pairs(recs), rn, lens)
    assert text == gzip.open(os.path.join(edges["d"], "hic_q0.pairs.gz")).read()
    assert_reaches_the_edges("hic_q0.pairs", text, dict(zip(edges["names"], lens)))
    assert m.format_pairs_gpu(m.postprocess_gpu(recs), rn, lens) == text


def _many_short_sequences(n_seq=70000, n_pairs=20000, seed=5):
    """n_seq sequences of 60 to 400 bp and 2x50 pairs, half of them on rids >= 2^16; every fragment lies inside its sequence."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    comp = np.zeros(256, dtype=np.uint8)
    comp[list(b"ACGT")] = list(b"TGCA")
    seqs = [acgt[rng.integers(0, 4, int(n))] for n in rng.integers(60, 401, n_seq)]
    names = ["scaffold_%d" % i for i in range(n_seq)]
    r1, r2 = [], []
    for p in range(n_pairs):
        rid = int(rng.integers(65536 if p % 2 else 0, n_seq))
        s = seqs[rid]
        if len(s) < 100:
            s = seqs[rid - 1] if len(seqs[rid - 1]) >= 100 else seqs[0]
        fl = int(rng.integers(50, len(s) + 1))
        st = int(rng.integers(0, len(s) - fl + 1))
        f = s[st:st + fl].copy()
        if rng.random() < 0.5:
            f[int(rng.integers(0, fl))] = acgt[rng.integers(0, 4)]
        a, b = f[:50].tobytes(), comp[f[-50:][::-1]].tobytes()
        if rng.random() < 0.5:
            a, b = b, a
        r1.append(a)
        r2.append(b)
    return seqs, names, pack(r1), pack(r2)


@pytest.fixture(scope="module")
def many(tmp_path_factory):
    seqs, names, (s1, o1), (s2, o2) = _many_short_sequences()
    path = str(tmp_path_factory.mktemp("many") / "ref.fa")
    with open(path, "wb") as f:
        for n, s in zip(names, seqs):
            f.write(b">" + n.encode() + b"\n" + s.tobytes() + b"\n")
    oref = orc.Reference(path)
    return dict(seqs=seqs, names=names, pairs=(s1, o1, s2, o2), oref=oref, oidx=orc.Index(ref=oref, k=17, w=7))


def test_many_short_sequences_index_mapping_and_bed_equal_oracle(many):
    m = cb.Mapper(cb.make_params("", max_read_length=64, mapq_threshold=0))
    m.upload_reference(many["seqs"], many["names"])
    m.build_index(17, 7)
    a, b = m.download_index(), many["oidx"].arrays()
    assert np.array_equal(a["occ"], b["occ"]) and len(a["occ"]) > 0
    s1, o1, s2, o2 = many["pairs"]
    recs, stats = m.map_batch(s1, o1, s2, o2)
    op = orc.make_params("", mapq_threshold=0)
    orecs, _ = orc.map_pairs(op, many["oidx"], many["oref"], s1, o1, s2, o2, n_threads=8)
    assert len(recs) == len(orecs) > 10000 and stats["n_overflow_pairs"] == 0
    assert_same_records(recs, orecs)
    assert (orecs["rid"] >= 65536).sum() > 3000
    want = orc.format_bed(many["oref"], orc.postprocess(op, orecs))
    assert m.format_bed(m.postprocess(recs)) == want
    assert m.format_bed_gpu(m.postprocess_gpu(recs)) == want


def test_many_short_sequences_pairs_equal_oracle(many):
    m = cb.Mapper(cb.make_params("hic", max_read_length=64, mapq_threshold=0))
    m.upload_reference(many["seqs"], many["names"])
    a = many["oidx"].arrays()
    m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    s1, o1, s2, o2 = many["pairs"]
    recs, stats = m.map_batch(s1, o1, s2, o2)
    orecs, _ = orc.map_pairs(orc.make_params("hic", mapq_threshold=0), many["oidx"], many["oref"], s1, o1, s2, o2, n_threads=8)
    assert len(recs) == len(orecs) > 10000 and stats["n_overflow_pairs"] == 0
    assert_same_records(recs, orecs)
    assert (orecs["rid1"] >= 65536).sum() > 3000
    rn = [b"p%d" % i for i in range(len(o1) - 1)]
    lens = [len(s) for s in many["seqs"]]
    text = m.format_pairs(m.postprocess_pairs(recs), rn, lens)
    assert text.count(b"\n") > 10000
    assert m.format_pairs_gpu(m.postprocess_gpu(recs), rn, lens) == text


@pytest.fixture(scope="module")
def cli_index(edges, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ix") / "edges.index")
    subprocess.check_call([CLI, "-i", "-r", os.path.join(edges["d"], "ref.fa.gz"), "-o", out], stderr=subprocess.DEVNULL)
    return out


# golden -> chromap-b200 arguments (make_golden_edges.sh)
CLI_ARGS = {"chip.bed": ["--preset", "chip"], "q0.bed": ["-q", "0"], "e15q0.bed": ["-e", "15", "-q", "0"], "e1q0.bed": ["-e", "1", "-q", "0"],
            "atac.bed": ["--preset", "atac"], "se_q0.bed": ["-q", "0"], "pe_q0.sam": ["--SAM", "-q", "0"], "se_q0.sam": ["--SAM", "-q", "0"],
            "hic_q0.pairs": ["--preset", "hic", "-q", "0"]}


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_cli_at_sequence_ends_equals_reference_binary_output(edges, cli_index, case, reader, tmp_path):
    assert sorted(CLI_ARGS) == sorted(EDGE_CASES)
    d = edges["d"]
    paired = EDGE_CASES[case][2]
    r1, r2 = ("hic_read1.fq.gz", "hic_read2.fq.gz") if case.startswith("hic") else ("read1.fq.gz", "read2.fq.gz")
    out = str(tmp_path / case)
    args = [CLI, "-x", cli_index, "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, r1)] + (["-2", os.path.join(d, r2)] if paired else [])
    r = subprocess.run(args + CLI_ARGS[case] + ["-o", out] + (["--host-reader"] if reader == "host" else []), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if reader == "device":
        assert "using the host reader" not in r.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(d, case + ".gz")).read()
