"""GPU parity at index shapes other than (17, 7) and at the mapping knobs the other GPU tests leave at their defaults: the CUDA
path (through the C ABI) against the CPU oracle and the reference binary's BEDs in tests/golden/synth_params.  Every shape but
(17, 7) runs the run-time minimizer scan (seed_front_kernel<false>); k > 22 keeps every minimizer in the record arrays.
Run with `-m gpu` on an H100."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.param_space import PARAM_CASES
from tests.test_gpu_parity import assert_same_records
from tests.util import load_pairs, read_fasta

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def synth(golden_dir):
    d = os.path.join(golden_dir, "synth_small")
    names, seqs = read_fasta(os.path.join(d, "ref.fa.gz"))
    oref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    return dict(d=d, out=os.path.join(golden_dir, "synth_params"), names=names, seqs=seqs, oref=oref, pairs=load_pairs(d), index={})


def _oindex(synth, k, w):
    if (k, w) not in synth["index"]:
        synth["index"][(k, w)] = orc.Index(ref=synth["oref"], k=k, w=w)
    return synth["index"][(k, w)]


def _mapper(synth, k, w, se, preset, kw, on_device, **extra):
    m = cb.Mapper(cb.make_params(preset, max_read_length=64, single_end=int(se), **dict(kw, **extra)))
    m.upload_reference(synth["seqs"], synth["names"])
    if on_device:
        m.build_index(k, w)
    else:
        a = _oindex(synth, k, w).arrays()
        m.upload_index(k, w, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
    info = m.index_info()
    assert (info["k"], info["w"]) == (k, w)
    return m


def _same_trace(tr, otrace):
    def same(f, mask):
        a, b = tr[f][mask], otrace[f][mask]
        if not np.array_equal(a, b):
            bad = np.nonzero(np.any(np.atleast_2d((a != b).T).T.reshape(len(a), -1), axis=1))[0][:5]
            raise AssertionError("%s differs at pairs %s: gpu %s oracle %s" % (f, np.nonzero(mask)[0][bad], a[bad], b[bad]))
    both = (otrace["n_minimizers"] > 0).all(axis=1)
    for f in ("n_minimizers", "trimmed_len", "n_pos_candidates_gen", "n_neg_candidates_gen", "supplement_result"):
        same(f, both)
    alive = otrace["n_records"] > 0
    for f in ("n_pos_candidates", "n_neg_candidates", "n_pos_mappings", "n_neg_mappings", "min_errors", "n_best",
              "min_sum_errors", "n_best_pairs", "n_second_best_pairs", "repetitive_seed_length", "trimmed_len"):
        same(f, alive)
    assert both.sum() > 3000 and alive.sum() > 1500


@pytest.mark.parametrize("on_device", [False, True], ids=["uploaded_index", "device_built_index"])
@pytest.mark.parametrize("case", sorted(PARAM_CASES))
def test_records_trace_and_bed_equal_oracle_and_golden(synth, case, on_device):
    k, w, se, preset, kw = PARAM_CASES[case]
    m = _mapper(synth, k, w, se, preset, kw, on_device)
    op = orc.make_params(preset, **kw)
    oidx = _oindex(synth, k, w)
    s1, o1, s2, o2 = synth["pairs"]
    if se:
        recs, stats = m.map_batch(s1, o1, None, None)
        orecs = orc.map_reads_se(op, oidx, synth["oref"], s1, o1)
    else:
        recs, stats = m.map_batch(s1, o1, s2, o2)
        orecs, otrace = orc.map_pairs(op, oidx, synth["oref"], s1, o1, s2, o2, trace=True)
        _same_trace(m.trace(len(o1) - 1), otrace)
    tiers = m.timing()["tier_pairs"]
    assert len(recs) == len(orecs) > 1500
    assert_same_records(recs, orecs)
    assert stats["n_overflow_pairs"] == 0
    if k > 22:  # the front end without its shared-memory key buffer handed records to seed_cta_kernel
        assert tiers[1] > 0, tiers
    want = gzip.open(os.path.join(synth["out"], case + ".bed.gz")).read()
    assert m.format_bed(m.postprocess(recs)) == want
    assert m.format_bed_gpu(m.postprocess_gpu(recs)) == want


def test_sam_cores_at_k23_w11_equal_oracle(synth):
    """output_format 4 (spans, CIGARs and MAPQ from those spans) on a (23, 11) index, e = 8."""
    m = _mapper(synth, 23, 11, False, "", {}, False, output_format=4)
    s1, o1, s2, o2 = synth["pairs"]
    recs, stats = m.map_batch(s1, o1, s2, o2)
    assert recs.dtype == cb.SAM_RECORD and stats["n_overflow_pairs"] == 0
    cores = orc.map_sam_cores(orc.make_params(""), _oindex(synth, 23, 11), synth["oref"], s1, o1, s2, o2)
    assert len(recs) == len(cores) > 1000
    for f in ("read_id", "rid", "mapq", "is_unique", "secondary", "overflow"):
        assert np.array_equal(recs[f], cores[f]), f
    for q in range(2):
        for f in ("pos", "end", "strand", "n_cigar"):
            bad = np.nonzero(recs[f][:, q] != cores[f][:, q])[0]
            assert len(bad) == 0, (f, q, bad[:5], recs[f][bad[:5], q], cores[f][bad[:5], q])
        for i in range(len(recs)):
            n = recs["n_cigar"][i, q]
            assert np.array_equal(recs["cigar"][i, q, :n], cores["cigar"][i, q, :n]), (i, q)


def test_heavy_repeats_at_k23_w11_equal_oracle(tmp_path):
    """100k pairs on 4 x 2 Mbp with planted repeats on a (23, 11) index built on the device: records == oracle, through the
    overflow tiers."""
    d = str(tmp_path)
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_synth.py"), "--out", d, "--seed", "29", "--n-seq", "4",
                           "--seq-len", "2000000", "--n-pairs", "100000", "--short-frac", "0.2"])
    names, seqs = read_fasta(os.path.join(d, "ref.fa"))
    oref = orc.Reference(os.path.join(d, "ref.fa"))
    oidx = orc.Index(ref=oref, k=23, w=11)
    s1, o1, s2, o2 = load_pairs(d, "read1.fq", "read2.fq")
    kw = dict(mapq_threshold=0, remove_pcr_duplicates=1)
    m = cb.Mapper(cb.make_params("", max_read_length=64, **kw))
    m.upload_reference(seqs, names)
    m.build_index(23, 11)
    assert np.array_equal(m.download_index()["occ"], oidx.arrays()["occ"])
    recs, stats = m.map_batch(s1, o1, s2, o2)
    tiers = m.timing()["tier_pairs"]
    orecs, _ = orc.map_pairs(orc.make_params("", **kw), oidx, oref, s1, o1, s2, o2, n_threads=8)
    assert stats["n_overflow_pairs"] == 0, tiers
    assert len(recs) == len(orecs) > 50000, tiers
    for f in recs.dtype.names:
        bad = np.nonzero(recs[f] != orecs[f])[0]
        assert len(bad) == 0, ("tier pairs %s" % tiers, f, bad[:5], recs[bad[:5]], orecs[bad[:5]])
    assert tiers[1] > 0, tiers
