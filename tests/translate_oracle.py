"""Test infrastructure: the reference's --barcode-translate restated for the oracle's barcoded BED writer.  SetTranslateTable,
ProcessTranslateFileLine and Translate (barcode_translator.h:42-145) as the writer uses them (mapping_writer.h:39-42,
mapping_writer.cc:18-24,131-137), on top of oracle/oracle_py.py; and the oracle's paired-end barcoded mapping with
--output-mappings-not-in-whitelist (orc_mapper_set_barcodes' last argument), which oracle_py.map_pairs_bc leaves off."""
import ctypes as C

import numpy as np

from oracle import oracle_py as orc


class TranslationUndefined(ValueError):
    """The reference's SetTranslateTable has no defined result for this table (see load_translation)."""


class BarcodeMissing(KeyError):
    """Translate's exit: "Barcode does not exist in the translation table." (barcode_translator.h:87-91)."""


def _seed(s):
    """GenerateSeedFromSequence (utils.h:111-129) over all of s: CharToUint8, an ambiguous base becomes A."""
    key = 0
    for c in s:
        key = (key << 2) | {65: 0, 97: 0, 67: 1, 99: 1, 71: 2, 103: 2, 84: 3, 116: 3}.get(c, 0)
    return key & 0xFFFFFFFFFFFFFFFF


def translation_lines(data):
    """The lines SetTranslateTable hands to ProcessTranslateFileLine (barcode_translator.h:42-68): gzgets into a 512-byte
    buffer (at most 511 bytes, up to and including a newline), one trailing newline removed, the rest cut at a NUL (the
    std::string is built from the C string)."""
    lines, i = [], 0
    while i < len(data):
        j = data.find(b"\n", i, i + 511)
        piece = data[i:j + 1] if j >= 0 else data[i:i + 511]
        i += len(piece)
        if piece.endswith(b"\n"):
            piece = piece[:-1]
        lines.append(piece.split(b"\0")[0])
    return lines


def load_translation(data):
    """SetTranslateTable + ProcessTranslateFileLine (barcode_translator.h:42-68,125-145) on a file's inflated bytes:
    {FROM key: TO bytes}, and from_bc_length_ from the last line.  Raises TranslationUndefined where the reference's result
    is undefined: no line (the mask shift count is negative), a line without FROM (GenerateSeedFromSequence with length -1),
    or from_bc_length_ >= 32 (the mask is a shift of 64 or more)."""
    table, from_len = {}, -1
    for line in translation_lines(data):
        i = next((k for k, c in enumerate(line) if c in b",\t"), len(line))
        from_len = len(line) - i - 1
        if from_len < 0:
            raise TranslationUndefined("a line without a separator")
        table[_seed(line[i + 1:])] = line[:i]  # kh_put: a repeated key takes the later value
    if from_len < 0 or from_len >= 32:
        raise TranslationUndefined("FROM length %d" % from_len)
    return table, from_len


def translate(translation, bc, bc_len):
    """Translate (barcode_translator.h:72-101): the TO strings of the bc_len / L segments joined by '-'."""
    table, L = translation
    mask = (1 << (2 * L)) - 1
    nseg = bc_len // L
    out = []
    for i in range(nseg):
        seed = (((int(bc) << (2 * i * L)) & 0xFFFFFFFFFFFFFFFF) >> (2 * (nseg - 1) * L)) & mask
        if seed not in table:
            raise BarcodeMissing(seed)
        out.append(table[seed])
    return b"-".join(out)


def format_bed_bc(ref, recs, bcs, bc_len, translation=None):
    """Barcoded BED text (mapping_writer.cc:127-137).  translation = load_translation(...): the barcode field goes through
    translate() (mapping_writer.cc:131-137); raises BarcodeMissing where the reference exits."""
    text = orc.format_bed_bc(ref, recs, bcs, bc_len)
    if translation is None:
        return text
    lines = text.split(b"\n")[:-1]
    out = []
    for line, bc in zip(lines, bcs):
        f = line.split(b"\t")
        f[3] = translate(translation, bc, bc_len)
        out.append(b"\t".join(f) + b"\n")
    return b"".join(out)


def map_pairs_bc(params, index, ref, seq1, off1, seq2, off2, barcodes, quals, bc_len, whitelist=None, first_read_id=0, n_threads=1,
                 output_not_in_whitelist=False):
    """oracle_py.map_pairs_bc with the whitelist's --output-mappings-not-in-whitelist flag."""
    L = orc.lib()
    m = L.orc_mapper_create(C.byref(params), index.h, ref.h)
    if whitelist is not None:
        L.orc_mapper_set_barcodes(m, whitelist.h, 1, 0.9, int(output_not_in_whitelist))
    n = len(off1) - 1
    out = np.zeros(n * params.max_num_best_mappings, dtype=orc.PE_RECORD)
    obc = np.zeros(len(out), dtype=np.uint64)
    st = np.zeros(2, dtype=np.uint64)
    seq1 = np.ascontiguousarray(seq1, dtype=np.uint8); seq2 = np.ascontiguousarray(seq2, dtype=np.uint8)
    off1 = np.ascontiguousarray(off1, dtype=np.uint32); off2 = np.ascontiguousarray(off2, dtype=np.uint32)
    barcodes = np.ascontiguousarray(barcodes, dtype=np.uint8); quals = np.ascontiguousarray(quals, dtype=np.uint8)
    got = L.orc_map_pairs_bc(m, n, seq1.ctypes.data, off1.ctypes.data, seq2.ctypes.data, off2.ctypes.data, barcodes.ctypes.data, quals.ctypes.data,
                             bc_len, first_read_id, out.ctypes.data, obc.ctypes.data, len(out), n_threads, st.ctypes.data)
    L.orc_mapper_free(m)
    return out[:got], obc[:got], st
