"""Builds and runs a host test of the device code: kernel headers of chromap_b200/csrc/, whole, compiled by g++ on top of the
host emulation of a CTA (tests/cta_emu.h), followed by the test's own main.  The headers go through file-wide syntactic
rewrites only; the spots that have no host form are left out by the headers themselves (#ifndef CMX_HOST_EMU)."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chromap_b200", "csrc")
ORACLE_H = os.path.join(ROOT, "oracle", "oracle_chromap.h")
ORACLE_LIB = os.path.join(ROOT, "oracle", "liboracle.so")

# the mapping pipeline, in include order
PIPELINE = ["device_common.cuh", "minimizers.cuh", "pipeline_kernels.cuh", "seed_front.cuh", "cta_pair_candidates.cuh", "cta_verify_pairing.cuh",
            "sam_kernels.cuh"]


def source(headers):
    """The headers as one host translation unit (without the shim)."""
    text = "\n".join(open(os.path.join(CSRC, h)).read() for h in headers)
    text = re.sub(r'#include [<"][^\n]*', "", text).replace("#pragma once", "")
    text = re.sub(r"#pragma unroll[^\n]*", "", text)
    text = re.sub(r"extern __shared__ (?:__align__\(\d+\) )?(\w+) (\w+)\[\];", r"\1 *\2 = (\1 *)g_dyn_smem;", text)
    return re.sub(r"asm volatile\(.*?\)\s*;", ";", text)   # the prefetch hints


def build(tmp_path, headers, main, sources=(), libs=(), flags=()):
    """Compiles cta_emu.h + the headers + main (C++ text) into tmp_path/t, linked to the oracle; returns the executable's path."""
    assert os.path.exists(ORACLE_LIB), "oracle/liboracle.so not built (__graft_entry__.build())"
    src = tmp_path / "t.cc"
    src.write_text('#include "%s"\n' % os.path.join(ROOT, "tests", "cta_emu.h") + source(headers) + main)
    exe = tmp_path / "t"
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-std=c++20", "-pthread", "-w"] + list(flags) + ["-o", str(exe), str(src)] + list(sources) +
                          [ORACLE_LIB, "-Wl,-rpath," + os.path.dirname(ORACLE_LIB), "-fopenmp"] + list(libs))
    return exe


def run(tmp_path, headers, main, args=(), timeout=1800, **kw):
    """build() and run the result; returns the subprocess.CompletedProcess (stdout / stderr as text)."""
    exe = build(tmp_path, headers, main, **kw)
    return subprocess.run([str(exe)] + list(args), capture_output=True, text=True, timeout=timeout)
