"""The oracle's bulk-level duplicate removal (tests/bulk_dedup_oracle.py: the low-memory merge loop transcribed over the oracle's
barcoded records) reproduces every file the reference binary wrote into tests/golden/synth_bulk_dedup, and the in-memory run,
where the level plays no part, with the oracle's cell-level post-processing."""
import hashlib
import os

import pytest

from tests import bulk_dedup_oracle as bdo


@pytest.mark.parametrize("name", sorted(bdo.RUNS))
def test_oracle_reproduces_golden(name):
    want = bdo.golden(name)
    md5 = dict(l.split()[::-1] for l in open(os.path.join(bdo.OUT, "md5.txt")))
    assert hashlib.md5(want).hexdigest() == md5[name + ".bed"]
    got = bdo.run(name)
    assert got.count(b"\n") == want.count(b"\n")
    assert got == want


def test_stats_count_the_lines():
    for l in open(os.path.join(bdo.OUT, "stats.txt")):
        f = l.split()
        assert bdo.golden(f[0][:-len(".bed")]).count(b"\n") == int(f[-1])
