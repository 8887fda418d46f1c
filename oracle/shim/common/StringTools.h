// Stand-in for the reference's common/StringTools.h when its core/common/Strptime.cpp is compiled in place
// (oracle/build_ref_strptime.sh): the one helper that translation unit calls.
#pragma once
#include <strings.h>

#include <string>

namespace logtail {
inline int CStringNCaseInsensitiveCmp(const char* s1, const char* s2, size_t n) { return strncasecmp(s1, s2, n); }
} // namespace logtail
