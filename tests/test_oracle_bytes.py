"""The CPU oracle against the reference binary on reads and a reference beyond upper-case ACGTN (tests/golden/synth_bytes,
make_golden_bytes.sh / tools/gen_bytes.py): a soft-masked reference with IUPAC codes and bytes 0x80-0xFF; reads that are wholly
or partly lower case or carry 'n', '.', IUPAC codes or bytes 0x60-0xDF opposite the reference's high bytes.  Several steps of
the reference compare raw bytes instead of case-folded base codes (the Hamming shortcut of the traceback, adapter trimming, the
Hi-C gap extension, SAM NM / MD and SEQ), so these inputs pin what case folding alone would not.
- every golden byte for byte;
- on normalised inputs (every byte CharToUint8 maps to a base as its upper-case base, every other byte as 'N'), the oracle's
  outputs differ from the decorated ones in exactly the line counts make_golden_bytes.sh recorded from the reference binary
  (stats.txt), and the counts that show the raw bytes at work stay above floors;
- a reference holding every byte 0x01-0xFF (but '\\n' and '\\r') inside random contexts: `chromap -i`, run here, and the oracle's
  index have the same content.
CPU only."""
import collections
import gzip
import hashlib
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_py as orc
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")

# name -> (preset, knobs, reads, paired, chromap-b200 / chromap options); make_golden_bytes.sh
CASES = {
    "chip.bed": ("chip", {}, "pe100", True, ["--preset", "chip"]),
    "q0.bed": ("", dict(mapq_threshold=0), "pe100", True, ["-q", "0"]),
    "atac.bed": ("atac", {}, "pe100", True, ["--preset", "atac"]),
    "chip.tagalign": ("chip", {}, "pe100", True, ["--preset", "chip", "--TagAlign"]),
    "q0.paf": ("", dict(mapq_threshold=0), "pe100", True, ["--PAF", "-q", "0"]),
    "pe_q0.sam": ("", dict(mapq_threshold=0), "pe100", True, ["--SAM", "-q", "0"]),
    "se_q0.sam": ("", dict(mapq_threshold=0), "pe100", False, ["--SAM", "-q", "0"]),
    "se_q0.bed": ("", dict(mapq_threshold=0), "pe100", False, ["-q", "0"]),
    "hic.pairs": ("hic", {}, "hic150", True, ["--preset", "hic"]),
    "hic_q0.pairs": ("hic", dict(mapq_threshold=0), "hic150", True, ["--preset", "hic", "-q", "0"]),
    "pe250_chip.bed": ("chip", {}, "pe250", True, ["--preset", "chip"]),
    "pe250_q0.sam": ("", dict(mapq_threshold=0), "pe250", True, ["--SAM", "-q", "0"]),
    "rf_rev.bed": ("chip", {}, "pe100", True, ["--preset", "chip", "--read-format", "r1:0:-1:-,r2:0:-1:-"]),
}
# outputs that must differ from the normalised run in at least this many lines (reads normalised, reference normalised, both):
# about half of what the reference binary showed.  Adapter trimming compares read 1 raw; SAM prints SEQ and MD from raw bytes.
DIFF_FLOORS = {"atac.bed": (50, 0, 50), "pe_q0.sam": (2200, 4000, 4500), "se_q0.sam": (1100, 2000, 2200), "pe250_q0.sam": (700, 1600, 1700)}

# CharToUint8 (utils.h): A/a C/c G/g T/t are bases, every other byte is 4
NORMALISE = np.full(256, ord("N"), dtype=np.uint8)
for _a, _b in zip(b"ACGTacgt", b"ACGTACGT"):
    NORMALISE[_a] = _b
# the complement --read-format's ':-' takes (utils.h:87-100): "ACGTNNNN"[3 ^ CharToUint8(c)], upper case
CUT_COMPLEMENT = np.full(256, ord("N"), dtype=np.uint8)
for _a, _b in zip(b"ACGTacgt", b"TGCATGCA"):
    CUT_COMPLEMENT[_a] = _b


def _write_fastq(path, text, f):
    """The FASTQ text with f applied to every sequence line (as a uint8 array)."""
    lines = text.split(b"\n")
    for i in range(1, len(lines), 4):
        lines[i] = f(np.frombuffer(lines[i], dtype=np.uint8)).tobytes()
    open(path, "wb").write(b"\n".join(lines))


def _write_fasta(path, text, f):
    open(path, "wb").write(b"\n".join(l if l[:1] == b">" else f(np.frombuffer(l, dtype=np.uint8)).tobytes() for l in text.split(b"\n")))


def make_inputs(d, out, reads=True, ref=True):
    """The synth_bytes inputs under out: uncompressed, with normalised reads and / or reference; plus the reads cut by rf_rev's
    --read-format (both mates reverse-complemented), and the oracle's index.  Returns out."""
    os.makedirs(out, exist_ok=True)
    keep = lambda a: a
    _write_fasta(os.path.join(out, "ref.fa"), gzip.open(os.path.join(d, "ref.fa.gz")).read(), NORMALISE.__getitem__ if ref else keep)
    for name in ("pe100", "hic150", "pe250"):
        for m in (1, 2):
            _write_fastq(os.path.join(out, "%s_%d.fq" % (name, m)), gzip.open(os.path.join(d, "%s_%d.fq.gz" % (name, m))).read(),
                         NORMALISE.__getitem__ if reads else keep)
    for m in (1, 2):
        _write_fastq(os.path.join(out, "rf_rev_%d.fq" % m), open(os.path.join(out, "pe100_%d.fq" % m), "rb").read(), lambda a: CUT_COMPLEMENT[a[::-1]])
    assert orc.Index(ref=orc.Reference(os.path.join(out, "ref.fa")), k=17, w=7).save(os.path.join(out, "ref.index")) == 0
    return out


def oracle_output(case, d, out):
    """The oracle's file for one case on the inputs under d (make_inputs), written to out; returns its bytes."""
    preset, kw, reads, paired, _ = CASES[case]
    p = orc.make_params(preset, **kw)
    if case == "rf_rev.bed":
        reads = "rf_rev"
    ref, index = os.path.join(d, "ref.fa"), os.path.join(d, "ref.index")
    r1, r2 = os.path.join(d, reads + "_1.fq"), os.path.join(d, reads + "_2.fq") if paired else None
    if case.endswith(".sam"):
        orc.run_files_sam(p, index, ref, r1, r2, out)
    elif case.endswith(".paf"):
        orc.run_files_paf(p, index, ref, r1, r2, out)
    elif case.endswith(".tagalign"):
        oref = orc.Reference(ref)
        recs, _ = orc.map_pairs(p, orc.Index(index), oref, *load_pairs(d, reads + "_1.fq", reads + "_2.fq"))
        open(out, "wb").write(orc.format_tagalign(oref, orc.postprocess(p, recs)))
    elif not paired:
        orc.run_files_se(p, index, ref, r1, out, 1)
    else:
        orc.run_files(p, index, ref, r1, r2, out)
    return open(out, "rb").read()


def line_diff(a, b):
    """Lines of a and b that the other lacks, as multisets (make_golden_bytes.sh's count)."""
    ca, cb = collections.Counter(a.splitlines()), collections.Counter(b.splitlines())
    return sum(((ca - cb) + (cb - ca)).values())


@pytest.fixture(scope="module")
def byte_set(golden_dir, tmp_path_factory):
    d = os.path.join(golden_dir, "synth_bytes")
    t = tmp_path_factory.mktemp("bytes")
    md5 = dict(reversed(line.split()) for line in open(os.path.join(d, "md5.txt")))
    stats = {f[0]: tuple(map(int, f[1:])) for f in (line.split() for line in open(os.path.join(d, "stats.txt")))}
    return dict(d=d, t=t, md5=md5, stats=stats, inputs=make_inputs(d, str(t / "raw"), reads=False, ref=False))


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_reproduces_reference_binary_on_raw_bytes(byte_set, tmp_path, case):
    want = gzip.open(os.path.join(byte_set["d"], case + ".gz")).read()
    assert hashlib.md5(want).hexdigest() == byte_set["md5"][case]
    assert want.count(b"\n") > 500
    assert oracle_output(case, byte_set["inputs"], str(tmp_path / case)) == want


def test_normalised_inputs_differ_in_the_recorded_lines(byte_set):
    s = byte_set
    assert sorted(s["stats"]) == sorted(CASES)
    dirs = [make_inputs(s["d"], str(s["t"] / n), reads=n != "ref", ref=n != "reads") for n in ("reads", "ref", "both")]
    got = {}
    for case in CASES:
        want = gzip.open(os.path.join(s["d"], case + ".gz")).read()
        got[case] = tuple(line_diff(want, oracle_output(case, d, os.path.join(d, "out." + case))) for d in dirs)
    assert got == s["stats"], got
    for case, floor in DIFF_FLOORS.items():
        assert all(g >= f for g, f in zip(got[case], floor)), (case, got[case], floor)


def all_bytes_reference(seed=47, copies=24, flank=30):
    """One sequence per line of flank random bases, one byte, flank random bases: every byte 0x01-0xFF but '\\n' and '\\r',
    `copies` times each, in a random order.  Returns the FASTA text and its sequences."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    mid = np.array([b for b in range(1, 256) if b not in (10, 13)] * copies, dtype=np.uint8)
    rng.shuffle(mid)
    units = np.concatenate([acgt[rng.integers(0, 4, (len(mid), flank))], mid[:, None], acgt[rng.integers(0, 4, (len(mid), flank))]], axis=1)
    seqs = [units[i:i + 2000].reshape(-1) for i in range(0, len(units), 2000)]
    text = b"".join(b">s%d\n" % i + b"\n".join(s[j:j + 2 * flank + 1].tobytes() for j in range(0, len(s), 2 * flank + 1)) + b"\n"
                    for i, s in enumerate(seqs))
    return text, seqs


def index_content(a):
    """(bucket count, occurrence table, occupied (key, value) pairs sorted): what a lookup can see of a khash index."""
    nb = a["n_buckets"]
    occupied = ((a["flags"][np.arange(nb) >> 4] >> ((np.arange(nb) & 15) << 1)) & 3) == 0
    kv = sorted(zip(a["keys"][occupied].tolist(), a["vals"][occupied].tolist()))
    return nb, a["occ"], kv


def test_oracle_index_on_every_byte_equals_reference_binary(tmp_path):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    text, seqs = all_bytes_reference()
    fa = tmp_path / "ref.fa"
    fa.write_bytes(text)
    subprocess.check_call([REF_BIN, "-i", "-r", str(fa), "-o", str(tmp_path / "ref.index")], stderr=subprocess.DEVNULL)
    ref = orc.Reference(str(fa))
    assert [bytes(ref.seq(i)) for i in range(ref.n)] == [s.tobytes() for s in seqs]
    theirs = index_content(orc.Index(str(tmp_path / "ref.index")).arrays())
    ours = index_content(orc.Index(ref=ref, k=17, w=7).arrays())
    assert theirs[0] == ours[0] and np.array_equal(theirs[1], ours[1]) and theirs[2] == ours[2]
    assert len(ours[2]) > 50000
