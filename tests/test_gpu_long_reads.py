"""Reads longer than 160 bases on the GPU path (tests/golden/synth_long, make_golden_long.sh).

Library: the same batches through a context created at the default 160 bases and grown by cmx_set_max_read_length, a
context created at the final length, and the oracle: identical records for BED, SAM cores, Hi-C pairs and single-end.
Beyond 320 bases (seeded reads, tests/long_reads_inputs.py): contexts of 416, 608 and 832 bases, one created at 843 (the
device bound), and mates of up to 1,400 bases at 832 through the overflow tiers.  Refused sizes leave the context as it was.
CLI: every golden with the device and the host reader; a run of two file sets, 2x50 then 2x250 (`-1 a,b`), so that the
context grows between them, and runs of 2x400, 2x832 and mates of 50 to 1,400 bases, each against the reference binary run
at test time; and a `--SAM` run that meets a 400-base read stops without writing its output file."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.long_reads_inputs import BEYOND_320_SETS, make_pairs, write_fastq, write_set
from tests.test_gpu_parity import assert_same_records
from tests.test_oracle_long import CASES
from tests.util import load_pairs, pack, read_fasta

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")


@pytest.fixture(scope="module")
def long_data(golden_dir):
    d = os.path.join(golden_dir, "synth_long")
    ref_path = os.path.join(golden_dir, "synth_sc", "ref.fa.gz")
    names, seqs = read_fasta(ref_path)
    oref = orc.Reference(ref_path)
    return dict(d=d, ref=ref_path, names=names, seqs=seqs, oref=oref, oidx=orc.Index(ref=oref, k=17, w=7),
                wl=os.path.join(golden_dir, "synth_sc", "whitelist.txt"))


def _mapper(data, preset, L, **kw):
    m = cb.Mapper(cb.make_params(preset, max_read_length=L, **kw))
    m.upload_reference(data["seqs"], data["names"])
    a = data["oidx"].arrays()
    m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    return m


def _same_sam_cores(recs, cores, paired):
    assert len(recs) == len(cores)
    for f in ("read_id", "rid", "mapq", "is_unique", "secondary", "overflow"):
        assert np.array_equal(recs[f], cores[f]), f
    for q in range(2 if paired else 1):
        for f in ("pos", "end", "strand", "n_cigar"):
            assert np.array_equal(recs[f][:, q], cores[f][:, q]), (f, q)
        for i in range(len(recs)):
            n = recs["n_cigar"][i, q]
            assert np.array_equal(recs["cigar"][i, q, :n], cores["cigar"][i, q, :n]), (i, q)


# reads -> final max_read_length; (output, preset, knobs)
LIB_CASES = {
    "pe250_chip": ("pe250", 256, "bed", "chip", {}),
    "pe300_atac": ("pe300", 320, "bed", "atac", {}),
    "mixed_q0": ("mixed", 320, "bed", "", dict(mapq_threshold=0)),
    "se250_chip": ("se250", 256, "bed", "chip", {}),
    "pe250_sam": ("pe250", 256, "sam", "", dict(mapq_threshold=0)),
    "se250_sam": ("se250", 256, "sam", "", dict(mapq_threshold=0)),
    "hic250": ("hic250", 256, "pairs", "hic", {}),
    "pe400_chip": ("pe400", 416, "bed", "chip", {}),
    "pe600_chip": ("pe600", 608, "bed", "chip", {}),
    "pe600_atac": ("pe600", 608, "bed", "atac", {}),
    "pe832_chip": ("pe832", 832, "bed", "chip", {}),
    "se600_chip": ("se600", 608, "bed", "chip", {}),
    "hic400": ("hic400", 416, "pairs", "hic", {}),
}


def _reads(data, reads):
    """(s1, o1, s2, o2) of a golden read set, or of a set beyond 320 bases drawn from its seed (s2 = o2 = None: single-end)."""
    if reads not in BEYOND_320_SETS:
        se = reads.startswith("se")
        s1, o1, s2, o2 = load_pairs(data["d"], reads + "_1.fq.gz", reads + "_1.fq.gz" if se else reads + "_2.fq.gz")
        return (s1, o1, None, None) if se else (s1, o1, s2, o2)
    pairs = make_pairs(reads, *BEYOND_320_SETS[reads])
    s1, o1 = pack([a for a, _ in pairs])
    if pairs[0][1] is None:
        return s1, o1, None, None
    s2, o2 = pack([b for _, b in pairs])
    return s1, o1, s2, o2


@pytest.mark.parametrize("case", sorted(LIB_CASES))
def test_grown_context_equals_created_context_and_oracle(long_data, case):
    reads, L, out, preset, kw = LIB_CASES[case]
    se = reads.startswith("se")
    kw = dict(kw, single_end=int(se), output_format=4 if out == "sam" else cb.make_params(preset).output_format)
    s1, o1, s2, o2 = _reads(long_data, reads)
    op = orc.make_params(preset, **{k: v for k, v in kw.items() if k != "output_format" or v != 4})  # the oracle's SAM cores take BED params
    grown = _mapper(long_data, preset, 160, **kw)
    before = None
    if out == "sam":  # at 160 bases the SAM cores of longer reads are reported as overflowed, not aligned
        with pytest.raises(cb.CmxError):
            grown.map_batch(s1, o1, s2, o2, first_read_id=7)
    elif L <= 4 * 160:  # every pair through the overflow tiers: the same records, only more slowly (the last tier takes 640 bases)
        before, _ = grown.map_batch(s1, o1, s2, o2, first_read_id=7)
    grown.set_max_read_length(L)
    created = _mapper(long_data, preset, L, **kw)
    got = [m.map_batch(s1, o1, s2, o2, first_read_id=7) for m in (grown, created)]
    for recs, stats in got:
        assert stats["n_overflow_pairs"] == 0 and len(recs) > (2000 if reads not in BEYOND_320_SETS else (len(o1) - 1) // 4)
    if out == "sam":
        cores = orc.map_sam_cores(op, long_data["oidx"], long_data["oref"], s1, o1, s2, o2, first_read_id=7)
        for recs, _ in got:
            _same_sam_cores(recs, cores, not se)
    else:
        if se:
            want = orc.map_reads_se(op, long_data["oidx"], long_data["oref"], s1, o1, first_read_id=7)
        else:
            want, _ = orc.map_pairs(op, long_data["oidx"], long_data["oref"], s1, o1, s2, o2, first_read_id=7)
        for recs, _ in got:
            assert_same_records(recs, want)
        if before is not None:
            assert_same_records(before, want)


def test_context_created_at_the_device_bound(long_data):
    """843 bases, the longest a context can be sized for (the front end's tiles then take 232,320 B of the 232,448 B of
    shared memory an H100 grants a CTA): 2x832 pairs stay out of the overflow tiers' refusal and map as the oracle does."""
    s1, o1, s2, o2 = _reads(long_data, "pe832")
    m = _mapper(long_data, "chip", 843)
    recs, stats = m.map_batch(s1, o1, s2, o2)
    print("tier pairs at 843:", m.timing()["tier_pairs"])
    assert stats["n_overflow_pairs"] == 0 and len(recs) > (len(o1) - 1) // 4
    want, _ = orc.map_pairs(orc.make_params("chip"), long_data["oidx"], long_data["oref"], s1, o1, s2, o2)
    assert_same_records(recs, want)


def test_mates_beyond_the_context_take_the_overflow_tiers(long_data):
    """Mates of 50 to 1,400 bases at 832: every pair with a mate over 832 bases goes to tier 1 (maxmm 1,664), and repeats of
    synth_sc's reference push some pairs on to tier 2 (maxmm 3,328), where the CTA kernels meet their largest shared-memory
    requests; the records are the oracle's."""
    s1, o1, s2, o2 = _reads(long_data, "mixed1400")
    n_long = int(np.sum((np.diff(o1) > 832) | (np.diff(o2) > 832)))
    m = _mapper(long_data, "chip", 832)
    recs, stats = m.map_batch(s1, o1, s2, o2)
    t = m.timing()["tier_pairs"]
    print("tier pairs at 832, mates of up to 1,400 bases:", t, "pairs with a mate over 832:", n_long)
    assert n_long > 100 and t[1] >= n_long and t[2] > 0 and stats["n_overflow_pairs"] == 0, t
    want, _ = orc.map_pairs(orc.make_params("chip"), long_data["oidx"], long_data["oref"], s1, o1, s2, o2)
    assert len(want) > 300
    assert_same_records(recs, want)


def test_grown_context_keeps_long_pairs_in_tier_0():
    """On a reference without repeats, 2x300 pairs all take the overflow tiers at 160 bases; grown to 320 (tier 0's hit
    capacity grows with the length too) nearly all of them stay in tier 0, with the oracle's records."""
    g = np.random.default_rng(3)
    seqs = [np.frombuffer(b"ACGT", dtype=np.uint8)[g.integers(0, 4, n)] for n in (1_500_000, 700_000)]
    names = ["r1", "r2"]
    pairs = make_pairs("pe300", 10000, 31, seqs)
    s1, o1 = pack([a for a, _ in pairs])
    s2, o2 = pack([b for _, b in pairs])
    oref = orc.Reference(seqs=seqs)
    oidx = orc.Index(ref=oref, k=17, w=7)
    m = _mapper(dict(seqs=seqs, names=names, oidx=oidx), "chip", 160)
    m.map_batch(s1, o1, s2, o2)
    assert m.timing()["tier_pairs"][:2] == [10000, 10000]
    m.set_max_read_length(320)
    recs, stats = m.map_batch(s1, o1, s2, o2)
    t = m.timing()["tier_pairs"]
    assert t[0] == 10000 and t[1] <= 100, t
    want, _ = orc.map_pairs(orc.make_params("chip"), oidx, oref, s1, o1, s2, o2)
    assert len(recs) > 9000
    assert_same_records(recs, want)


def test_refused_sizes_leave_the_context_usable(long_data):
    s1, o1, s2, o2 = load_pairs(long_data["d"], "pe250_1.fq.gz", "pe250_2.fq.gz")
    m = _mapper(long_data, "", 160, output_format=4, mapq_threshold=0)
    for bad in (29, 352, 1601):  # below min_read_length, SAM beyond 320, beyond the verification bound
        with pytest.raises(cb.CmxError):
            m.set_max_read_length(bad)
    m.set_max_read_length(256)
    with pytest.raises(cb.CmxError):
        m.set_max_read_length(321)
    recs, stats = m.map_batch(s1, o1, s2, o2)
    _same_sam_cores(recs, orc.map_sam_cores(orc.make_params("", mapq_threshold=0), long_data["oidx"], long_data["oref"], s1, o1, s2, o2), True)
    b = _mapper(long_data, "chip", 160)
    for bad in (1601, 844):  # beyond the verification bound; front-end tiles beyond an H100's 227 KB of shared memory
        with pytest.raises(cb.CmxError):
            b.set_max_read_length(bad)
    b.set_max_read_length(832)  # the longest the command line sizes for
    recs, stats = b.map_batch(s1, o1, s2, o2)
    want, _ = orc.map_pairs(orc.make_params("chip"), long_data["oidx"], long_data["oref"], s1, o1, s2, o2)
    assert_same_records(recs, want)


@pytest.fixture(scope="module")
def cli_data(long_data, tmp_path_factory):
    if not os.path.exists(CLI):
        import __graft_entry__
        __graft_entry__.build()
    t = tmp_path_factory.mktemp("long_cli")
    ref = str(t / "ref.fa")
    with open(ref, "wb") as f:
        f.write(gzip.open(long_data["ref"]).read())
    idx = str(t / "ref.index")
    subprocess.check_call([CLI, "-i", "-r", ref, "-o", idx], stderr=subprocess.DEVNULL)
    return dict(t=t, ref=ref, idx=idx)


def _cli_args(case, d, wl):
    preset, kw, reads = CASES[case]
    a = ["--preset", preset] if preset else []
    if kw.get("mapq_threshold") == 0:
        a += ["-q", "0"]
    if case.endswith(".sam"):
        a.append("--SAM")
    if case.endswith(".tagalign"):
        a.append("--TagAlign")
    a += ["-1", os.path.join(d, reads + "_1.fq.gz")]
    if not reads.startswith("se"):
        a += ["-2", os.path.join(d, reads + "_2.fq.gz")]
    if "_sc_" in case:
        a += ["-b", os.path.join(d, "barcode.fq.gz"), "--barcode-whitelist", wl]
    return a


@pytest.mark.parametrize("case,reader", [(c, r) for c in sorted(CASES) for r in ("device", "host") if not (r == "device" and c.endswith(".sam"))])
def test_cli_equals_reference_on_long_reads(long_data, cli_data, case, reader):
    """Every golden; --SAM reads on the host whatever the option says."""
    out = str(cli_data["t"] / ("%s.%s" % (reader, case)))
    args = [CLI, "-x", cli_data["idx"], "-r", cli_data["ref"], "-o", out] + _cli_args(case, long_data["d"], long_data["wl"])
    if reader == "host":
        args.append("--host-reader")
    p = subprocess.run(args, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    assert "mapping scratch resized for" in p.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(long_data["d"], case + ".gz")).read()


@pytest.mark.parametrize("reader", ["device", "host"])
def test_cli_grows_between_file_sets_like_the_reference(cli_data, reader):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    t = cli_data["t"]
    a1, a2 = write_set(str(t), "pe50", 3000, 50, tag="set_a")
    b1, b2 = write_set(str(t), "pe250", 3000, 2500, tag="set_b")
    args = ["--preset", "chip", "-x", cli_data["idx"], "-r", cli_data["ref"], "-1", a1 + "," + b1, "-2", a2 + "," + b2]
    want, got = str(t / "ref_two_sets.bed"), str(t / ("%s_two_sets.bed" % reader))
    subprocess.check_call([REF_BIN, "-t", "1", "-o", want] + args, stderr=subprocess.DEVNULL)
    p = subprocess.run([CLI, "-o", got] + args + (["--host-reader"] if reader == "host" else []), capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stderr.count("mapping scratch resized for 256-base reads") == 1
    w = open(want, "rb").read()
    assert w.count(b"\n") > 3000 and open(got, "rb").read() == w


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("kind,resized", [("pe400", 416), ("pe832", 832), ("mixed1400", 832)])
def test_cli_equals_reference_beyond_320_bases(cli_data, kind, resized, reader):
    """2x400, 2x832 and mates of 50 to 1,400 bases (the context stops at 832; longer mates take the overflow tiers)."""
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    t = cli_data["t"]
    r1, r2 = write_set(str(t), kind, *BEYOND_320_SETS[kind])
    args = ["--preset", "chip", "-x", cli_data["idx"], "-r", cli_data["ref"], "-1", r1, "-2", r2]
    want, got = str(t / ("ref_%s.bed" % kind)), str(t / ("%s_%s.bed" % (reader, kind)))
    if not os.path.exists(want):
        subprocess.check_call([REF_BIN, "-t", "1", "-o", want] + args, stderr=subprocess.DEVNULL)
    p = subprocess.run([CLI, "-o", got] + args + (["--host-reader"] if reader == "host" else []), capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stderr.count("mapping scratch resized for %d-base reads" % resized) == 1, p.stderr[-2000:]
    w = open(want, "rb").read()
    assert w.count(b"\n") > 300 and open(got, "rb").read() == w


def test_cli_sam_refuses_reads_longer_than_320_before_writing(cli_data):
    t = cli_data["t"]
    r = write_set(str(t), "pe250", 200, 9, tag="with400")
    reads = [l for l in gzip.open(r[0]).read().split(b"\n")[1::4]]
    reads[150] = reads[150] + reads[151][:150]  # one 400-base read in the middle of the file
    write_fastq(r[0], reads, "with400.")
    out = str(t / "with400.sam")
    p = subprocess.run([CLI, "--SAM", "-x", cli_data["idx"], "-r", cli_data["ref"], "-1", r[0], "-2", r[1], "-o", out], capture_output=True, text=True)
    assert p.returncode != 0 and "up to 320 bases" in p.stderr and "400 bases" in p.stderr, p.stderr[-1000:]
    assert not os.path.exists(out)
