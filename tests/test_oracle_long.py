"""The CPU oracle against the reference binary's outputs on reads longer than 160 bases (tests/golden/synth_long,
make_golden_long.sh): 2x250 and 2x300 pairs, mates of 50 to 300 bases, single-end 250, Hi-C-like 2x250, in BED (chip,
atac with adapter trimming, barcoded atac), TagAlign, SAM and pairs.  Beyond 320 bases, up to the 832 the command line sizes
for and mates of up to 1,400 bases, against the reference binary (oracle/_ref/chromap) run at test time on seeded reads.
Every file byte for byte.  CPU only."""
import gzip
import hashlib
import os
import subprocess

import pytest

from oracle import oracle_py as orc
from tests.long_reads_inputs import BEYOND_320_SETS, write_set
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")

# name -> (preset, knobs, reads)
CASES = {
    "pe250_chip.bed": ("chip", {}, "pe250"),
    "pe300_chip.bed": ("chip", {}, "pe300"),
    "mixed_chip.bed": ("chip", {}, "mixed"),
    "se250_chip.bed": ("chip", {}, "se250"),
    "pe250_atac.bed": ("atac", {}, "pe250"),
    "pe300_atac.bed": ("atac", {}, "pe300"),
    "pe250_chip.tagalign": ("chip", {}, "pe250"),
    "pe250_q0.sam": ("", dict(mapq_threshold=0), "pe250"),
    "mixed_q0.sam": ("", dict(mapq_threshold=0), "mixed"),
    "se250_q0.sam": ("", dict(mapq_threshold=0), "se250"),
    "pe250_sc_atac.bed": ("atac", {}, "pe250"),
    "hic250.pairs": ("hic", {}, "hic250"),
}
# beyond 320 bases (BEYOND_320_SETS); SAM stays at 320 bases or fewer, where the GPU path writes it
BEYOND_320 = {
    "pe400_chip.bed": ("chip", {}, "pe400"),
    "pe600_chip.bed": ("chip", {}, "pe600"),
    "pe832_chip.bed": ("chip", {}, "pe832"),
    "mixed1400_chip.bed": ("chip", {}, "mixed1400"),
    "pe600_atac.bed": ("atac", {}, "pe600"),
    "pe832_atac.bed": ("atac", {}, "pe832"),
    "pe400_chip.tagalign": ("chip", {}, "pe400"),
    "se600_chip.bed": ("chip", {}, "se600"),
    "hic400.pairs": ("hic", {}, "hic400"),
}


@pytest.fixture(scope="module")
def long_set(golden_dir, tmp_path_factory):
    d = os.path.join(golden_dir, "synth_long")
    ref_path = os.path.join(golden_dir, "synth_sc", "ref.fa.gz")
    p = str(tmp_path_factory.mktemp("long") / "ref.index")
    assert orc.Index(ref=orc.Reference(ref_path), k=17, w=7).save(p) == 0
    md5 = dict(reversed(line.split()) for line in open(os.path.join(d, "md5.txt")))
    return dict(d=d, ref=ref_path, index=p, md5=md5, wl=os.path.join(golden_dir, "synth_sc", "whitelist.txt"))


def oracle_output(case, s, out, cases=CASES):
    """The oracle's file for one case, written to out."""
    preset, kw, reads = cases[case]
    d = s["d"]
    p = orc.make_params(preset, **kw)
    r1 = os.path.join(d, reads + "_1.fq.gz")
    r2 = None if reads.startswith("se") else os.path.join(d, reads + "_2.fq.gz")
    if case.endswith(".sam"):
        orc.run_files_sam(p, s["index"], s["ref"], r1, r2, out)
    elif case.endswith(".tagalign"):
        ref = orc.Reference(s["ref"])
        idx = orc.Index(ref=ref, k=17, w=7)
        recs, _ = orc.map_pairs(p, idx, ref, *load_pairs(d, reads + "_1.fq.gz", reads + "_2.fq.gz"))
        open(out, "wb").write(orc.format_tagalign(ref, orc.postprocess(p, recs)))
    elif "_sc_" in case:
        orc.run_files_bc(p, s["index"], s["ref"], r1, r2, os.path.join(d, "barcode.fq.gz"), s["wl"], out)
    elif r2 is None:
        orc.run_files_se(p, s["index"], s["ref"], r1, out, 1)
    else:
        orc.run_files(p, s["index"], s["ref"], r1, r2, out)
    return open(out, "rb").read()


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_reproduces_reference_binary_on_long_reads(long_set, tmp_path, case):
    want = gzip.open(os.path.join(long_set["d"], case + ".gz")).read()
    assert hashlib.md5(want).hexdigest() == long_set["md5"][case]
    assert want.count(b"\n") > 2500
    assert oracle_output(case, long_set, str(tmp_path / case)) == want


@pytest.fixture(scope="module")
def beyond_320_set(golden_dir, tmp_path_factory):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    t = tmp_path_factory.mktemp("beyond_320")
    ref_gz = os.path.join(golden_dir, "synth_sc", "ref.fa.gz")
    ref_fa = str(t / "ref.fa")
    open(ref_fa, "wb").write(gzip.open(ref_gz).read())
    ref_index, index = str(t / "ref.index"), str(t / "oracle.index")
    subprocess.check_call([REF_BIN, "-i", "-r", ref_fa, "-o", ref_index], stderr=subprocess.DEVNULL)
    assert orc.Index(ref=orc.Reference(ref_gz), k=17, w=7).save(index) == 0
    for kind, (n, seed) in BEYOND_320_SETS.items():
        write_set(str(t), kind, n, seed)
    return dict(d=str(t), ref=ref_gz, ref_fa=ref_fa, ref_index=ref_index, index=index)


def reference_binary_args(case, d):
    """The reference binary's options (and chromap-b200's) for one BEYOND_320 case, its reads under d."""
    preset, kw, reads = BEYOND_320[case]
    a = ["--preset", preset] + (["--TagAlign"] if case.endswith(".tagalign") else []) + ["-1", os.path.join(d, reads + "_1.fq.gz")]
    return a if reads.startswith("se") else a + ["-2", os.path.join(d, reads + "_2.fq.gz")]


@pytest.mark.parametrize("case", sorted(BEYOND_320))
def test_oracle_reproduces_reference_binary_beyond_320_bases(beyond_320_set, tmp_path, case):
    s = beyond_320_set
    want_path = str(tmp_path / ("ref." + case))
    subprocess.check_call([REF_BIN, "-t", "1", "-x", s["ref_index"], "-r", s["ref_fa"], "-o", want_path] + reference_binary_args(case, s["d"]),
                          stderr=subprocess.DEVNULL)
    want = open(want_path, "rb").read()
    assert want.count(b"\n") > 300
    assert oracle_output(case, s, str(tmp_path / case), BEYOND_320) == want
