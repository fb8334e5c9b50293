"""The CPU oracle at index shapes other than (17, 7) and at the mapping knobs the other goldens leave at their defaults, against
the reference binary's BEDs in tests/golden/synth_params (make_golden_params.sh).  CPU only."""
import gzip
import hashlib
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_py as orc
from tests.param_space import PARAM_CASES
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")


@pytest.fixture(scope="module")
def synth(golden_dir):
    d = os.path.join(golden_dir, "synth_small")
    oref = orc.Reference(os.path.join(d, "ref.fa.gz"))
    md5 = dict(reversed(line.split()) for line in open(os.path.join(golden_dir, "synth_params", "md5.txt")))
    return dict(d=d, out=os.path.join(golden_dir, "synth_params"), oref=oref, pairs=load_pairs(d), md5=md5, index={})


def _index(synth, k, w):
    if (k, w) not in synth["index"]:
        synth["index"][(k, w)] = orc.Index(ref=synth["oref"], k=k, w=w)
    return synth["index"][(k, w)]


@pytest.mark.parametrize("case", sorted(PARAM_CASES))
def test_oracle_reproduces_reference_bed_across_index_shapes_and_knobs(synth, case):
    k, w, se, preset, kw = PARAM_CASES[case]
    p = orc.make_params(preset, **kw)
    idx = _index(synth, k, w)
    assert (idx.k, idx.w) == (k, w)
    s1, o1, s2, o2 = synth["pairs"]
    if se:
        bed = orc.format_bed(synth["oref"], orc.postprocess_se(p, orc.map_reads_se(p, idx, synth["oref"], s1, o1)))
    else:
        recs, _ = orc.map_pairs(p, idx, synth["oref"], s1, o1, s2, o2)
        bed = orc.format_bed(synth["oref"], orc.postprocess(p, recs))
    want = gzip.open(os.path.join(synth["out"], case + ".bed.gz")).read()
    assert hashlib.md5(want).hexdigest() == synth["md5"][case + ".bed"]
    assert want.count(b"\n") > 1500
    assert bed == want


def _occupied(a):
    nb = a["n_buckets"]
    return ((a["flags"][np.arange(nb) >> 4] >> ((np.arange(nb) & 15) << 1)) & 3) == 0


@pytest.mark.parametrize("k,w", [(19, 10), (23, 11), (28, 20)])
def test_oracle_index_equals_reference_binary_index(synth, tmp_path, k, w):
    """`chromap -i -k K -w W` on synth_small and the oracle's builder: the same bucket count, the same occurrence table byte for
    byte, and the same key -> value map (the bucket order inside khash's arrays follows its resize history, not the content)."""
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    path = str(tmp_path / "ref.index")
    r = subprocess.run([REF_BIN, "-i", "-k", str(k), "-w", str(w), "-r", os.path.join(synth["d"], "ref.fa.gz"), "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-500:]
    theirs = orc.Index(path)
    assert (theirs.k, theirs.w) == (k, w)
    a, b = theirs.arrays(), _index(synth, k, w).arrays()
    assert a["n_buckets"] == b["n_buckets"]
    assert len(a["occ"]) > 0 and np.array_equal(a["occ"], b["occ"])
    oa, ob = _occupied(a), _occupied(b)
    ka, va, kb, vb = a["keys"][oa], a["vals"][oa], b["keys"][ob], b["vals"][ob]
    assert len(ka) == len(kb) > 10000
    ia, ib = np.argsort(ka), np.argsort(kb)
    assert np.array_equal(ka[ia], kb[ib]) and np.array_equal(va[ia], vb[ib])
