// Regular expression -> byte DFA, on the host (PQ_OP_REGEX).  The semantics restate the regex crate as arrow-string's
// regexp_is_match uses it (an unanchored search: TRUE when some substring matches); include/parseable_b200.h lists the
// syntax, the refusals and the limits.  The DFA it writes is what regex_match.cuh walks.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace pqb {

// Hard caps: a pattern is outside input, so a pathological one must end in an error, never in a hang or an OOM.
constexpr size_t kRxMaxPattern = 64 * 1024;        // bytes of pattern
constexpr uint32_t kRxMaxNfa = 65536;              // Thompson NFA states
constexpr uint32_t kRxMaxDfa = 4096;               // DFA states (dead and matched included)
constexpr size_t kRxMaxTable = 1u << 20;           // bytes of transition table
constexpr uint32_t kRxMaxNest = 250;               // nesting of groups and repetitions

// Compile `pat` (UTF-8, not NUL-terminated).  `case_insensitive` is the flag `i` from the start.  Returns 0 and the DFA blob
// (layout in regex_match.cuh), or PQ_ERR_INVALID_ARG (-1) / PQ_ERR_UNSUPPORTED (-2) with a message that names the byte
// position in the pattern.
int regex_compile(const char* pat, size_t n, bool case_insensitive, std::vector<uint8_t>& blob, std::string& err);

}  // namespace pqb
