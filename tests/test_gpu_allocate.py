"""--allocate-multi-mappings on the H100: cmx_allocate_multi_mappings_gpu against its host twin and the oracle's restatement
(tests/allocate_oracle.h) field by field, on the golden data sets and on a heavy-repeat set mapped on the device; its refusals;
and chromap-b200 end to end against every output of the reference binary (tests/golden/synth_allocate), log counts included."""
import gzip
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import chromap_b200 as cb
from chromap_b200.binding import AllocationStats
from oracle import oracle_py as orc
from tests import allocate_oracle as ao
from tests.test_cli import _ensure_cli
from tests.util import load_pairs, read_fasta

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def alloc_lib(tmp_path_factory):
    return ao.load(tmp_path_factory.mktemp("alloc_oracle"))


def _mapper(oparams):
    p = cb.make_params("")
    for f, _ in orc.Params._fields_:
        setattr(p, f, getattr(oparams, f))
    return cb.Mapper(p, device=0)


def _same(a, b):
    assert len(a) == len(b)
    for f in a.dtype.names:
        assert np.array_equal(a[f], b[f]), f


def _three_ways(m, lib, p, recs, keys, n_seq, distance, seed):
    gr, gk, gs = m.allocate_multi_mappings_gpu(recs, keys, distance, seed)
    hr, hk, hs = m.allocate_multi_mappings(recs, keys, distance, seed)
    orr, okk, ost = ao.allocate(lib, p, recs, keys, n_seq, distance, seed)
    _same(gr, hr); _same(gr, orr)
    if keys is not None:
        assert np.array_equal(gk, hk) and np.array_equal(gk, okk)
    assert gs == hs
    assert {f: gs[f] for f in ost} == ost
    return gr, gk, gs


@pytest.mark.parametrize("case", sorted(ao.CASES))
def test_abi_equals_host_twin_oracle_and_golden(case, alloc_lib, golden_dir):
    c = ao.CASES[case]
    ref, p, recs, keys, bc_len = ao.oracle_records(golden_dir, case)
    gr, gk, gs = _three_ways(_mapper(p), alloc_lib, p, recs, keys, ref.n, c["distance"], c["seed"])
    d = os.path.join(golden_dir, "synth_allocate")
    assert ao.format_text(ref, case, gr, gk, bc_len) == gzip.open(os.path.join(d, case + "." + c["fmt"] + ".gz")).read()
    want = ao.golden_stats(os.path.join(d, "stats.txt"))[case]
    assert {f: gs[f] for f in want} == want


def test_heavy_repeats_n8_several_seeds_and_distances(alloc_lib, tmp_path):
    """100k pairs on 4 x 2 Mbp with planted repeats (tools/gen_synth.py --seed 29), mapped on the device at -n 8 -q 0."""
    d = str(tmp_path)
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_synth.py"), "--out", d, "--seed", "29", "--n-seq", "4",
                           "--seq-len", "2000000", "--n-pairs", "100000", "--short-frac", "0.2"])
    names, seqs = read_fasta(os.path.join(d, "ref.fa"))
    s1, o1, s2, o2 = load_pairs(d, "read1.fq", "read2.fq")
    kw = dict(max_num_best_mappings=8, mapq_threshold=0)
    m = cb.Mapper(cb.make_params("", max_read_length=64, **kw))
    m.upload_reference(seqs, names)
    m.build_index(17, 7)
    recs, _ = m.map_batch(s1, o1, s2, o2)
    p = orc.make_params("", **kw)
    draws = 0
    for seed, dist in ((11, 0), (5, 200), (-1, 5000), (0, 2 ** 31 - 1)):
        _, _, gs = _three_ways(m, alloc_lib, p, recs, None, len(names), dist, seed)
        draws += gs["n_draws"]
        assert gs["n_multi"] > 20000 and gs["n_allocated"] > 1000, gs
    assert draws > 10000


def test_no_multi_mapping_and_low_memory_are_refused(golden_dir):
    ref, p, recs, _, _ = ao.oracle_records(golden_dir, "q0")
    few = np.ascontiguousarray(recs[recs["read_id"] < 3])
    assert len(few) and (few["mapq"] >= 4).all()
    m = _mapper(p)
    buf = few.copy()
    n, st = cb.binding.C.c_uint64(), AllocationStats()
    for fn in (m.L.cmx_allocate_multi_mappings_gpu, m.L.cmx_allocate_multi_mappings):
        rc = fn(m.h, buf.ctypes.data, None, len(buf), 0, 11, cb.binding.C.byref(n), cb.binding.C.byref(st))
        assert rc == -3 and b"aborts" in m.L.cmx_last_error(m.h)
        assert buf.tobytes() == few.tobytes()
    lm = cb.Mapper(cb.make_params("chip"), device=0)
    with pytest.raises(cb.CmxError, match="low-memory"):
        lm.allocate_multi_mappings_gpu(recs)
    with pytest.raises(cb.CmxError, match="distance -1"):
        m.allocate_multi_mappings_gpu(recs, distance=-1)


def test_records_without_any_uni_mapping_give_an_empty_output(alloc_lib, golden_dir):
    """Every record multi (mapq < 4): no read has a uni-mapping to overlap, all are dropped; CMX_OK with nothing left, as the
    reference and the host twin."""
    ref, p, recs, _, _ = ao.oracle_records(golden_dir, "n4q0")
    recs = recs.copy()
    recs["mapq"] %= 4
    m = _mapper(p)
    for dist in (0, 5000):
        gr, _, gs = _three_ways(m, alloc_lib, p, recs, None, ref.n, dist, 11)
        assert len(gr) == 0 and gs["n_multi"] > 1000 and gs["n_allocated"] == 0 and gs["n_without_overlap"] > 0, gs
        assert gs["n_uni_after"] == gs["n_multi_after"] == 0


@pytest.fixture(scope="module")
def cli_index(tmp_path_factory, golden_dir):
    cli = _ensure_cli()
    out = {}
    for data in ("synth_small", "synth_sc"):
        idx = str(tmp_path_factory.mktemp("idx") / "ref.index")
        subprocess.check_call([cli, "-i", "-r", os.path.join(golden_dir, data, "ref.fa.gz"), "-o", idx], stderr=subprocess.DEVNULL)
        out[data] = idx
    return out


def _cli_files(golden_dir, c, idx):
    d = os.path.join(golden_dir, c["data"])
    a = ["-x", idx, "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "read1.fq.gz")]
    if not c["se"]:
        a += ["-2", os.path.join(d, "read2.fq.gz")]
    if c["bc"]:
        a += ["-b", os.path.join(d, "barcode.fq.gz"), "--barcode-whitelist", os.path.join(d, "whitelist.txt")]
    return a


@pytest.mark.parametrize("reader", [[], ["--host-reader"]])
@pytest.mark.parametrize("case", sorted(ao.CASES))
def test_cli_reproduces_reference_binary(case, reader, cli_index, golden_dir, tmp_path):
    c = ao.CASES[case]
    out = str(tmp_path / ("out." + c["fmt"]))
    r = subprocess.run([_ensure_cli(), "--allocate-multi-mappings"] + c["args"] + reader + _cli_files(golden_dir, c, cli_index[c["data"]]) + ["-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    d = os.path.join(golden_dir, "synth_allocate")
    assert open(out, "rb").read() == gzip.open(os.path.join(d, case + "." + c["fmt"] + ".gz")).read()
    want = ao.golden_stats(os.path.join(d, "stats.txt"))[case]
    got = ao.golden_stats_text("== %s\n%s" % (case, r.stderr))[case]
    assert got == want


@pytest.mark.parametrize("preset", ["chip", "atac"])
def test_cli_low_memory_presets_ignore_the_option(preset, cli_index, golden_dir, tmp_path):
    d = os.path.join(golden_dir, "synth_small")
    out = str(tmp_path / "out.bed")
    subprocess.check_call([_ensure_cli(), "--preset", preset, "--allocate-multi-mappings", "--multi-mapping-allocation-seed", "3", "-x", cli_index["synth_small"],
                           "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "read1.fq.gz"), "-2", os.path.join(d, "read2.fq.gz"), "-o", out],
                          stderr=subprocess.DEVNULL)
    assert open(out, "rb").read() == gzip.open(os.path.join(d, preset + ".bed.gz")).read()


def test_cli_low_memory_sam_and_hic_ignore_the_option(cli_index, golden_dir, tmp_path):
    """Low-memory runs accept --allocate-multi-mappings with any output, SAM and Hi-C pairs included, and never allocate."""
    cli = _ensure_cli()
    d = os.path.join(golden_dir, "synth_small")
    base = ["-x", cli_index["synth_small"], "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "read1.fq.gz")]
    pe = base + ["-2", os.path.join(d, "read2.fq.gz")]
    out = str(tmp_path / "out.sam")
    subprocess.check_call([cli, "--preset", "chip", "--SAM", "--allocate-multi-mappings"] + pe + ["-o", out], stderr=subprocess.DEVNULL)
    assert open(out, "rb").read() == gzip.open(os.path.join(d, "pe_chip.sam.gz")).read()
    texts = []
    for extra in ([], ["--allocate-multi-mappings", "--multi-mapping-allocation-distance", "-7"]):
        out = str(tmp_path / ("lm%d.sam" % len(extra)))
        subprocess.check_call([cli, "--low-mem", "--SAM", "-n", "3", "-q", "0"] + extra + base + ["-o", out], stderr=subprocess.DEVNULL)
        texts.append(open(out, "rb").read())
    assert texts[0] == texts[1] and texts[0].count(b"\n") > 1000
    h = os.path.join(golden_dir, "synth_hic")
    idx = str(tmp_path / "hic.index")
    subprocess.check_call([cli, "-i", "-r", os.path.join(h, "ref.fa.gz"), "-o", idx], stderr=subprocess.DEVNULL)
    out = str(tmp_path / "out.pairs")
    subprocess.check_call([cli, "--preset", "hic", "--allocate-multi-mappings", "-x", idx, "-r", os.path.join(h, "ref.fa.gz"), "-1", os.path.join(h, "read1.fq.gz"),
                           "-2", os.path.join(h, "read2.fq.gz"), "-o", out], stderr=subprocess.DEVNULL)
    assert open(out, "rb").read() == gzip.open(os.path.join(h, "hic.pairs.gz")).read()


def test_cli_without_multi_mappings_fails_and_writes_nothing(cli_index, golden_dir, tmp_path):
    d = os.path.join(golden_dir, "synth_small")
    fq = []
    for r in ("read1", "read2"):
        p = str(tmp_path / (r + ".fq"))
        open(p, "wb").write(b"".join(gzip.open(os.path.join(d, r + ".fq.gz")).readlines()[:12]))
        fq.append(p)
    out = str(tmp_path / "out.bed")
    r = subprocess.run([_ensure_cli(), "--allocate-multi-mappings", "-q", "0", "-x", cli_index["synth_small"], "-r", os.path.join(d, "ref.fa.gz"),
                        "-1", fq[0], "-2", fq[1], "-o", out], capture_output=True, text=True)
    assert r.returncode != 0 and "the reference aborts here" in r.stderr and not os.path.exists(out), r.stderr[-1000:]
