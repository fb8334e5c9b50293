"""`chromap-b200` with several read files per option: `-1`, `-2` and `-b` take comma-separated lists and quoted glob patterns,
expanded before any device work.  These are the outcomes decided while the options are read, so no GPU is needed."""
import os
import shutil
import subprocess

import pytest

from tests.test_cli import _ensure_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "tests", "golden", "ref_test")


def _run(tmp_path, reads):
    cli = _ensure_cli()
    return subprocess.run([cli, "-x", os.path.join(D, "ref.index"), "-r", os.path.join(D, "ref.fa.gz")] + reads + ["-o", str(tmp_path / "never.bed")],
                          capture_output=True, text=True)


@pytest.fixture
def lanes(tmp_path):
    """Two lanes of read 1 / read 2 / barcode files, named as a sequencer names them."""
    for lane in ("L001", "L002"):
        shutil.copy(os.path.join(D, "read1.fq"), str(tmp_path / ("s_%s_R1.fq" % lane)))
        shutil.copy(os.path.join(D, "read2.fq"), str(tmp_path / ("s_%s_R2.fq" % lane)))
        shutil.copy(os.path.join(D, "read1.fq"), str(tmp_path / ("s_%s_I1.fq" % lane)))
    return tmp_path


def test_shorter_read2_or_barcode_list_is_refused(lanes):
    p = lambda name: str(lanes / name)
    r = _run(lanes, ["-1", p("s_L001_R1.fq") + "," + p("s_L002_R1.fq"), "-2", p("s_L001_R2.fq")])
    assert r.returncode == 255 and "-2 lists 1 file(s), -1 lists 2" in r.stderr, r.stderr
    r = _run(lanes, ["-1", p("s_L00*_R1.fq"), "-2", p("s_L00*_R2.fq"), "-b", p("s_L001_I1.fq")])
    assert r.returncode == 255 and "-b lists 1 file(s), -1 lists 2" in r.stderr, r.stderr
    assert "no CPU fallback" not in r.stderr


def test_pattern_without_match_is_refused(lanes):
    r = _run(lanes, ["-1", str(lanes / "s_L00*_R1.fq"), "-2", str(lanes / "s_L00*_R3.fq")])
    assert r.returncode == 255 and "no file matches " + str(lanes / "s_L00*_R3.fq") in r.stderr, r.stderr
    r = _run(lanes, ["-1", str(lanes / "s_L001_R1.fq") + "," + str(lanes / "missing.fq"), "-2", str(lanes / "s_L001_R2.fq")])
    assert r.returncode == 255 and "Cannot find sequence file " + str(lanes / "missing.fq") in r.stderr, r.stderr
    assert "no CPU fallback" not in r.stderr


def test_lists_and_patterns_reach_the_device(lanes):
    """A comma list and a glob that resolve are accepted, their files listed in order, and the run goes on to the device;
    -2 files beyond the -1 files are never read, with a warning."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the mapping runs are in test_gpu_cli_files")
    p = lambda name: str(lanes / name)
    comma = ["-1", p("s_L001_R1.fq") + "," + p("s_L002_R1.fq"), "-2", p("s_L001_R2.fq") + "," + p("s_L002_R2.fq"), "-b", p("s_L001_I1.fq") + "," + p("s_L002_I1.fq")]
    glob = ["-1", p("s_L00?_R1.fq"), "-2", p("s_L00[12]_R2.fq"), "-b", p("s_*_I1.fq")]
    for reads in (comma, glob):
        r = _run(lanes, reads)
        assert r.returncode != 0 and "no CPU fallback" in r.stderr, r.stderr
        listed = [l for l in r.stderr.splitlines() if l.startswith(str(lanes))]
        assert listed == [p("s_L001_R1.fq"), p("s_L002_R1.fq"), p("s_L001_R2.fq"), p("s_L002_R2.fq"), p("s_L001_I1.fq"), p("s_L002_I1.fq")], r.stderr
    r = _run(lanes, ["-1", p("s_L001_R1.fq"), "-2", p("s_L00*_R2.fq")])
    assert r.returncode != 0 and "no CPU fallback" in r.stderr, r.stderr
    assert "WARNING: -2 lists 2 file(s), -1 lists 1: the last 1 file(s) of -2 are not read." in r.stderr
