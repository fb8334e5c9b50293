"""chromap-b200 --allocate-multi-mappings: the refusals that need no device (a negative distance; SAM, PAF and pairs output in an
in-memory run), and the low-memory runs that accept the option (they then stop at the missing device like any run here).
CPU only."""
import os
import subprocess

from tests.test_cli import _ensure_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "tests", "golden", "ref_test")
FILES = ["-x", os.path.join(D, "ref.index"), "-r", os.path.join(D, "ref.fa.gz"), "-1", os.path.join(D, "read1.fq"), "-2", os.path.join(D, "read2.fq")]


def _run(args, tmp_path):
    out = str(tmp_path / "never.out")
    r = subprocess.run([_ensure_cli()] + args + FILES + ["-o", out], capture_output=True, text=True)
    return r, os.path.exists(out)


def test_negative_distance_is_refused(tmp_path):
    r, wrote = _run(["--allocate-multi-mappings", "--multi-mapping-allocation-distance", "-1"], tmp_path)
    assert r.returncode != 0 and "--multi-mapping-allocation-distance -1: use 0 or more" in r.stderr and not wrote


def test_sam_paf_pairs_are_refused_in_memory(tmp_path):
    for fmt in (["--SAM"], ["--PAF"], ["--split-alignment", "--pairs"]):
        r, wrote = _run(fmt + ["--allocate-multi-mappings", "-q", "0"], tmp_path)
        assert r.returncode != 0 and "not with --SAM, --PAF or --pairs" in r.stderr and not wrote, (fmt, r.stderr)


def test_options_parse_and_low_memory_runs_accept_them(tmp_path):
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("with a device these runs map: test_gpu_allocate.py runs them against the goldens")
    for args in (["--allocate-multi-mappings", "--multi-mapping-allocation-distance", "200", "--multi-mapping-allocation-seed", "-1"],
                 ["--preset", "chip", "--allocate-multi-mappings", "--multi-mapping-allocation-distance", "-5"],
                 ["--preset", "hic", "--allocate-multi-mappings"], ["--low-mem", "--SAM", "--allocate-multi-mappings"]):
        r, wrote = _run(args, tmp_path)
        assert r.returncode != 0 and "no CPU fallback" in r.stderr and not wrote, (args, r.stderr)
        assert "Will allocate multi-mappings after mapping." in r.stderr


def test_help_lists_the_options():
    r = subprocess.run([_ensure_cli(), "--help"], capture_output=True, text=True)
    for o in ("--allocate-multi-mappings", "--multi-mapping-allocation-distance", "--multi-mapping-allocation-seed"):
        assert o in r.stdout
