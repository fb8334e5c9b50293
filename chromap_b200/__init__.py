"""chromap_b200 — H100-native (sm_90a) replacement for Chromap's per-read mapping hot path.

Thin ctypes view of the C ABI in include/chromap_b200.h (chromap_b200/libchromap_b200.so, built by
`__graft_entry__.build()` / chromap_b200/csrc/Makefile).  There is no CPU fallback: importing works
anywhere, but creating a Mapper without the CUDA library or without a GPU raises.
"""
from .binding import (Mapper, Params, PE_RECORD, PAIRS_RECORD, PAIR_TRACE, SAM_RECORD, Timing, CmxError, lib_path, load_library,
                      make_params, taskloop_chunks, format_sam, format_sam_bc, format_paf, exchange_finish, ExchangeStats, ReadRange,
                      parse_read_format, apply_read_range, BarcodeTranslation, BarcodeNotTranslated, parse_barcode_translation,
                      format_bed_bc_tr)

__all__ = ["format_sam", "format_sam_bc", "format_paf", "Mapper", "Params", "PE_RECORD", "PAIRS_RECORD", "PAIR_TRACE", "SAM_RECORD", "Timing", "CmxError", "lib_path", "load_library",
           "make_params", "taskloop_chunks", "exchange_finish", "ExchangeStats", "ReadRange", "parse_read_format", "apply_read_range",
           "BarcodeTranslation", "BarcodeNotTranslated", "parse_barcode_translation", "format_bed_bc_tr"]
