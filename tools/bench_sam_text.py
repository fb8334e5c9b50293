"""Time of the SAM writer on the device (cmx_format_sam_gpu) against its host twin (cmx_format_sam_bc) on barcoded paired-end
lines: the SAM cores and barcode keys cmx_map_batch_pe gives for tests/golden/synth_sam_bc's pe_q0dedup run (synth_sc, -q 0,
--remove-pcr-duplicates), replicated with their reads (new read ids, other cells) to at least --lines lines.  Each call is host
memory in and out into a buffer of the text's size, so the time includes the copies over PCIe; it is a host clock around calls
that return after the device is done.  The median of --reps calls of each; the two texts are compared.  Prints one JSON line
with the card's name and power limit beside the times.

    python tools/bench_sam_text.py [--lines N] [--reps R] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import chromap_b200 as cb  # noqa: E402
from chromap_b200.binding import _sam_read_set  # noqa: E402
from tests import sam_bc_oracle as sbo  # noqa: E402
from tests.sam_bc_device import device_cores as _device_cores, reads as _reads  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    m, seqs, cores, keys, bc_len = _device_cores("pe_q0dedup")
    _, _, r1, r2 = sbo.setup()
    reps = -(-a.lines // (2 * len(cores)))
    n_reads = len(r1)
    big = np.concatenate([cores] * reps)
    big["read_id"] += np.repeat(np.arange(reps, dtype=np.uint32) * n_reads, len(cores))
    bk = np.concatenate([keys] * reps) ^ np.repeat(np.arange(reps, dtype=np.uint64) << 8, len(cores))
    reads1 = tuple(x * reps for x in _reads(r1))
    reads2 = tuple(x * reps for x in _reads(r2))
    keep = []
    rs1, rs2 = _sam_read_set(reads1, keep), _sam_read_set(reads2, keep)
    L = cb.load_library()
    names = (C.c_char_p * len(m.names))(*[s.encode() for s in m.names])
    lens = np.array([len(s) for s in seqs], dtype=np.uint32)
    concat = np.concatenate(seqs).astype(np.uint8)
    roff = np.zeros(len(seqs) + 1, dtype=np.uint64)
    roff[1:] = np.cumsum(lens.astype(np.uint64))
    big = np.ascontiguousarray(big); bk = np.ascontiguousarray(bk)
    dev = lambda buf, cap: L.cmx_format_sam_gpu(m.h, names, lens.ctypes.data, len(seqs), big.ctypes.data, bk.ctypes.data, bc_len, len(big), C.byref(rs1),
                                                C.byref(rs2), 0, buf, cap)
    host = lambda buf, cap: L.cmx_format_sam_bc(C.byref(m.params), names, lens.ctypes.data, len(seqs), concat.ctypes.data, roff.ctypes.data, big.ctypes.data,
                                                bk.ctypes.data, bc_len, len(big), C.byref(rs1), C.byref(rs2), 0, None, buf, cap)
    n = dev(None, 0)
    assert n > 0, n
    res = {"cores": len(big), "lines": None, "bytes": int(n), "card": card(), "reps": a.reps}
    for label, f in (("device", dev), ("host", host)):
        buf = C.create_string_buffer(n + 1)
        times = []
        for _ in range(a.reps + (1 if label == "device" else 0)):  # the device's first call warms up (module load, allocations)
            t0 = time.perf_counter()
            assert f(buf, n) == n
            times.append(time.perf_counter() - t0)
        if label == "device":
            times = times[1:]
            text = buf.raw[:n]
            res["lines"] = text.count(b"\n") - len(seqs)
        else:
            res["texts_equal"] = buf.raw[:n] == text
        res[label] = {"seconds_median": float(np.median(times)), "seconds_min": float(min(times))}
    res["speedup_median"] = res["host"]["seconds_median"] / res["device"]["seconds_median"]
    m.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
