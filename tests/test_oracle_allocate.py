"""--allocate-multi-mappings: the oracle's mapping, its in-memory post-processing and the allocation restatement of
tests/allocate_oracle.h reproduce every output of the unmodified reference binary (tests/golden/make_golden_allocate.sh) byte for
byte, and the counts of its log lines.  CPU only."""
import gzip
import hashlib
import os

import pytest

from tests import allocate_oracle as ao


@pytest.fixture(scope="module")
def alloc_lib(tmp_path_factory):
    return ao.load(tmp_path_factory.mktemp("alloc_oracle"))


def _md5s(d):
    return dict(reversed(line.split()) for line in open(os.path.join(d, "md5.txt")))


@pytest.mark.parametrize("case", sorted(ao.CASES))
def test_oracle_allocation_reproduces_reference_binary(case, alloc_lib, golden_dir):
    d = os.path.join(golden_dir, "synth_allocate")
    c = ao.CASES[case]
    ref, p, recs, keys, bc_len = ao.oracle_records(golden_dir, case)
    got = ao.allocate(alloc_lib, p, recs, keys, ref.n, c["distance"], c["seed"])
    assert got is not None
    r, k, stats = got
    name = case + "." + c["fmt"]
    want = gzip.open(os.path.join(d, name + ".gz")).read()
    assert hashlib.md5(want).hexdigest() == _md5s(d)[name]
    assert ao.format_text(ref, case, r, k, bc_len) == want
    gs = ao.golden_stats(os.path.join(d, "stats.txt"))[case]
    assert {f: stats[f] for f in gs} == gs


def test_oracle_refuses_a_run_without_multi_mappings(alloc_lib, golden_dir):
    """The first three pairs of synth_small map uniquely: the reference aborts there, the restatement reports it."""
    c = "q0"
    ref, p, recs, keys, _ = ao.oracle_records(golden_dir, c)
    few = recs[recs["read_id"] < 3]
    assert len(few) and (few["mapq"] >= 4).all()
    assert ao.allocate(alloc_lib, p, few, None, ref.n) is None
