// chromap_b200 host side — --read-format ranges (read_range.cc)
#pragma once
#include "../../../include/chromap_b200.h"

namespace cmxhost {

// 1..CMX_MAX_READ_RANGES ranges, 0 <= start <= end, ascending and disjoint, -1 in the last one only
bool ReadRangeRepresentable(const cmx_read_range &r);
// the whole read on the forward strand: no cut at all
inline bool ReadRangeIsWhole(const cmx_read_range &r) { return r.n == 1 && r.start[0] == 0 && r.end[0] == -1 && !r.reverse; }

}  // namespace cmxhost
