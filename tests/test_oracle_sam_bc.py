"""The oracle's barcoded SAM (tests/sam_bc_oracle.py: the barcode gate in front of orc_map_sam_cores, SAMMapping's order and
duplicate test with the cell barcode, CB:Z:) reproduces every file the reference binary wrote into tests/golden/synth_sam_bc."""
import gzip
import hashlib
import os

import pytest

from tests import sam_bc_oracle as sbo


@pytest.mark.parametrize("name", sorted(sbo.RUNS))
def test_oracle_reproduces_golden(name):
    want = gzip.open(os.path.join(sbo.OUT, name + ".sam.gz")).read()
    md5 = dict(l.split()[::-1] for l in open(os.path.join(sbo.OUT, "md5.txt")))
    assert hashlib.md5(want).hexdigest() == md5[name + ".sam"]
    got = sbo.run(name)
    assert got.count(b"\n") == want.count(b"\n")
    assert got == want
