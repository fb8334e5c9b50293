"""Test infrastructure: a context set up for one run of tests/sam_bc_oracle.RUNS (the synth_sc reference and index, the run's
whitelist) and the SAM cores and barcode keys cmx_map_batch_pe gives for it.  Needs a GPU; used by the GPU tests and
tools/bench_sam_text.py."""
import os

import numpy as np

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests import sam_bc_oracle as sbo
from tests.util import read_fasta

SC = sbo.SC


def params(name):
    preset, kw, se, _, _, _, _, _ = sbo.RUNS[name]
    return cb.make_params(preset, output_format=4, single_end=int(se), **kw)


def mapper(name):
    """A context for the run: the synth_sc reference and index, the run's whitelist."""
    names, seqs = read_fasta(os.path.join(SC, "ref.fa.gz"))
    m = cb.Mapper(params(name))
    m.upload_reference(seqs, names)
    m.build_index(17, 7)
    _, _, _, bc_path, wl_path, err, notinwl, _ = sbo.RUNS[name]
    bcs, quals, bc_len = sbo.bce.read_barcodes(bc_path if os.path.isabs(bc_path) else os.path.join(SC, bc_path))
    if wl_path:
        wl = orc.Whitelist(wl_path, bc_len)
        wl.sample(bcs)
        keys, counts, ns = wl.arrays()
        m.upload_barcode_whitelist(keys, counts, ns, bc_len, err, 0.9, notinwl)
    return m, seqs, bcs, quals, bc_len


def reads(recs):
    return [r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs]


def device_cores(name):
    m, seqs, bcs, quals, bc_len = mapper(name)
    _, _, r1, r2 = sbo.setup()
    se = sbo.RUNS[name][2]
    s1, o1 = pack([r[1] for r in r1])
    s2, o2 = (None, None) if se else pack([r[1] for r in r2])
    cores, st = m.map_batch(s1, o1, s2, o2, barcodes=bcs, barcode_quals=quals, bc_len=bc_len)
    return m, seqs, cores, st["barcode_keys"], bc_len


def pack(reads):
    off = np.zeros(len(reads) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(r) for r in reads])
    return np.frombuffer(b"".join(reads), dtype=np.uint8), off
