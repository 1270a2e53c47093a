// Regular expression -> byte DFA (see regex_compile.hpp, and include/parseable_b200.h for the semantics).
//
// 1. parse the pattern into an AST whose leaves are code point sets (literals, `.`, classes: case orbits already applied)
//    and assertions;
// 2. Thompson NFA over BYTES: a code point set becomes UTF-8 byte-range sequences (the usual range splitting), with
//    shared suffixes;
// 3. an implicit byte-level `.*?` loop in front (the search is unanchored);
// 4. subset construction over byte equivalence classes.  `^` / `$` under `m` are look-behind / look-ahead on `\n`: a DFA
//    state remembers whether the previous byte was `\n` (or the text started) when it still holds an unresolved
//    look-ahead, and a transition resolves look-aheads with the byte it consumes.  A state that has reached a match is
//    replaced by the absorbing matched state: a match test needs nothing after that.
//
// The `.*?` prefix is a loop over every byte, so it may put the pattern's start in the middle of a code point.  That adds no
// match: every path of the pattern's automaton consumes whole UTF-8 sequences, so its first byte is an ASCII or a lead
// byte, never a continuation byte, and a path that consumes bytes can only start on a code point boundary of valid UTF-8
// (arrow Utf8 is valid UTF-8).  A path that consumes no byte matches the empty string, which its assertions decide: `\A`,
// `^` and `\z`, `$` look at the text's ends and at `\n`, and any position next to those is a code point boundary.
#include "regex_compile.hpp"

#include <algorithm>
#include <cstring>
#include <map>
#include <memory>

#include "regex_match.cuh"

namespace pqb {
namespace {

#include "regex_unicode.inc"

struct RxError {
  int code;
  std::string msg;
};
[[noreturn]] void fail(int code, size_t pos, const std::string& what) {
  throw RxError{code, "regular expression: " + what + " at byte " + std::to_string(pos)};
}
[[noreturn]] void too_large(const char* what) {
  throw RxError{-2, std::string("regular expression too large for the device DFA: ") + what};
}
constexpr int kInvalid = -1, kUnsupported = -2;
constexpr uint32_t kMaxCp = 0x10FFFF;

// ---- code point sets ----
using Ranges = std::vector<std::pair<uint32_t, uint32_t>>;   // inclusive, sorted and merged after norm()

void norm(Ranges& r) {
  std::sort(r.begin(), r.end());
  Ranges o;
  for (auto& x : r) {
    if (!o.empty() && x.first <= o.back().second + 1) o.back().second = std::max(o.back().second, x.second);
    else o.push_back(x);
  }
  r.swap(o);
}
Ranges negate(const Ranges& r) {   // over the scalar values (surrogates are never in a set: utf8_seqs drops them)
  Ranges o;
  uint32_t lo = 0;
  for (auto& x : r) {
    if (x.first > lo) o.push_back({lo, x.first - 1});
    lo = x.second + 1;
  }
  if (lo <= kMaxCp) o.push_back({lo, kMaxCp});
  return o;
}
template <size_t N>
Ranges table(const uint32_t (&t)[N][2]) {
  Ranges r;
  for (size_t i = 0; i < N; i++) r.push_back({t[i][0], t[i][1]});
  return r;
}
// simple case folding: add every orbit member of every code point in the set
void case_fold(Ranges& r) {
  constexpr size_t nf = sizeof(kRxFold) / sizeof(kRxFold[0]);
  auto find = [](uint32_t c) {
    return std::lower_bound(kRxFold, kRxFold + nf, c, [](const uint32_t (&e)[2], uint32_t v) { return e[0] < v; });
  };
  Ranges add;
  for (auto& x : r)
    for (auto* e = find(x.first); e != kRxFold + nf && (*e)[0] <= x.second; ++e)
      for (uint32_t c = (*e)[1]; c != (*e)[0];) {   // the orbit is a cycle through the table
        add.push_back({c, c});
        auto* f = find(c);
        if (f == kRxFold + nf || (*f)[0] != c) break;
        c = (*f)[1];
      }
  r.insert(r.end(), add.begin(), add.end());
  norm(r);
}

// ---- AST ----
enum NodeKind { N_EMPTY, N_SET, N_ASSERT, N_CONCAT, N_ALT, N_REPEAT };
enum AssertKind : uint32_t { A_START_TEXT, A_END_TEXT, A_START_LINE, A_END_LINE };
struct Node {
  NodeKind kind;
  Ranges set;
  uint32_t akind = 0;
  uint32_t min = 0, max = 0;   // N_REPEAT; max == ~0u: unbounded
  std::vector<std::unique_ptr<Node>> kids;
  explicit Node(NodeKind k) : kind(k) {}
};
using P = std::unique_ptr<Node>;

struct Flags {
  bool i = false, m = false, s = false;
};

class Parser {
 public:
  Parser(const uint8_t* p, size_t n) : p_(p), n_(n) {}
  P parse(Flags f) {
    P r = alternation(f, 0);
    if (pos_ < n_) fail(kInvalid, pos_, "unopened group ')'");   // alternation only stops early at ')'
    return r;
  }

 private:
  const uint8_t* p_;
  size_t n_;
  size_t pos_ = 0;
  std::vector<std::string> names_;

  bool eof() const { return pos_ >= n_; }
  uint32_t peek() const { return p_[pos_]; }

  // one UTF-8 code point of the pattern
  uint32_t cp() {
    const size_t at = pos_;
    const uint32_t b = p_[pos_++];
    if (b < 0x80) return b;
    int k = b >= 0xF0 && b <= 0xF4 ? 3 : b >= 0xE0 ? (b <= 0xEF ? 2 : -1) : (b >= 0xC2 ? 1 : -1);
    if (k < 0 || pos_ + k > n_) fail(kInvalid, at, "pattern is not valid UTF-8");
    uint32_t c = b & (0x3Fu >> k);
    for (int j = 0; j < k; j++) {
      const uint32_t t = p_[pos_++];
      if ((t & 0xC0) != 0x80) fail(kInvalid, at, "pattern is not valid UTF-8");
      c = (c << 6) | (t & 0x3F);
    }
    const uint32_t minv[] = {0, 0x80, 0x800, 0x10000};
    if (c < minv[k] || c > kMaxCp || (c >= 0xD800 && c <= 0xDFFF)) fail(kInvalid, at, "pattern is not valid UTF-8");
    return c;
  }

  static P set_node(Ranges r, const Flags& f) {
    P n(new Node(N_SET));
    if (f.i) case_fold(r);
    else norm(r);
    n->set = std::move(r);
    return n;
  }

  P alternation(Flags f, uint32_t depth) {
    if (depth > kRxMaxNest) fail(kUnsupported, pos_, "nested too deeply");
    std::vector<P> alts;
    alts.push_back(concat(f, depth));
    while (!eof() && peek() == '|') {
      pos_++;
      alts.push_back(concat(f, depth));
    }
    if (alts.size() == 1) return std::move(alts[0]);
    P n(new Node(N_ALT));
    n->kids = std::move(alts);
    return n;
  }

  // `f` is shared by the rest of the group: a flag group `(?i)` changes it for what follows, across `|` too
  P concat(Flags& f, uint32_t depth) {
    P n(new Node(N_CONCAT));
    bool last_repeatable = false;
    uint32_t stacked = 0;   // quantifiers stacked on the last item (`a**`): each one nests
    while (!eof() && peek() != '|' && peek() != ')') {
      const size_t at = pos_;
      const uint32_t c = peek();
      if (c == '*' || c == '+' || c == '?' || c == '{') {
        if (!last_repeatable) fail(kInvalid, at, "repetition operator missing expression");
        uint32_t mn, mx;
        pos_++;
        if (c == '*') { mn = 0; mx = ~0u; }
        else if (c == '+') { mn = 1; mx = ~0u; }
        else if (c == '?') { mn = 0; mx = 1; }
        else counted(at, mn, mx);
        if (!eof() && peek() == '?') pos_++;   // lazy: the same match test
        P r(new Node(N_REPEAT));
        r->min = mn;
        r->max = mx;
        r->kids.push_back(std::move(n->kids.back()));
        n->kids.back() = std::move(r);
        if (depth + ++stacked > kRxMaxNest) fail(kUnsupported, at, "nested too deeply");
        continue;
      }
      P a = atom(f, depth);
      last_repeatable = a != nullptr;
      stacked = 0;
      if (a) n->kids.push_back(std::move(a));
    }
    if (n->kids.empty()) return P(new Node(N_EMPTY));
    return n;
  }

  uint32_t decimal(size_t at) {
    const size_t s = pos_;
    uint64_t v = 0;
    while (!eof() && peek() >= '0' && peek() <= '9') {
      v = v * 10 + (peek() - '0');
      if (v > 0xFFFFFFFFull) fail(kInvalid, at, "invalid repetition count");
      pos_++;
    }
    if (pos_ == s) fail(kInvalid, at, "invalid repetition count: expected a decimal");
    return uint32_t(v);
  }
  void counted(size_t at, uint32_t& mn, uint32_t& mx) {
    if (eof()) fail(kInvalid, at, "unclosed counted repetition");
    if (peek() == ',') fail(kUnsupported, at, "counted repetition {,m}");
    mn = decimal(at);
    mx = mn;
    if (!eof() && peek() == ',') {
      pos_++;
      if (!eof() && peek() == '}') mx = ~0u;
      else mx = decimal(at);
    }
    if (eof() || peek() != '}') fail(kInvalid, at, "unclosed counted repetition");
    pos_++;
    if (mx != ~0u && mn > mx) fail(kInvalid, at, "invalid counted repetition: min > max");
  }

  // nullptr: a flag group (nothing to repeat)
  P atom(Flags& f, uint32_t depth) {
    const size_t at = pos_;
    const uint32_t c = peek();
    switch (c) {
      case '(': return group(f, depth);
      case '[': {
        pos_++;
        Ranges r = bracket(f, at);
        P n(new Node(N_SET));
        n->set = std::move(r);
        return n;
      }
      case '.': {
        pos_++;
        Ranges r;
        if (f.s) r.push_back({0, kMaxCp});
        else { r.push_back({0, 9}); r.push_back({11, kMaxCp}); }
        P n(new Node(N_SET));
        n->set = r;
        return n;
      }
      case '^': case '$': {
        pos_++;
        P n(new Node(N_ASSERT));
        n->akind = c == '^' ? (f.m ? A_START_LINE : A_START_TEXT) : (f.m ? A_END_LINE : A_END_TEXT);
        return n;
      }
      case '\\': {
        pos_++;
        if (eof()) fail(kInvalid, at, "incomplete escape sequence");
        const uint32_t e = peek();
        if (e == 'A' || e == 'z') {
          pos_++;
          P n(new Node(N_ASSERT));
          n->akind = e == 'A' ? A_START_TEXT : A_END_TEXT;
          return n;
        }
        Ranges r;
        escape(at, r, false);
        return set_node(std::move(r), f);
      }
      default: {
        Ranges r{{cp(), 0}};
        r[0].second = r[0].first;
        return set_node(std::move(r), f);
      }
    }
  }

  // after '\': one escape as a code point set.  in_class: inside [...]
  void escape(size_t at, Ranges& r, bool in_class) {
    const uint32_t e = peek();
    if (e >= 0x80) fail(kInvalid, at, "unrecognized escape sequence");
    pos_++;
    auto one = [&](uint32_t v) { r.push_back({v, v}); };
    switch (e) {
      case 't': one('\t'); return;
      case 'n': one('\n'); return;
      case 'r': one('\r'); return;
      case 'f': one('\f'); return;
      case 'v': one('\v'); return;
      case 'a': one(7); return;
      case 'x': one(hex(at, 2)); return;
      case 'u': one(hex(at, 4)); return;
      case 'U': one(hex(at, 8)); return;
      case 'd': case 'D': case 's': case 'S': case 'w': case 'W': {
        Ranges t = e == 'd' || e == 'D' ? table(kRxDigit) : e == 's' || e == 'S' ? table(kRxSpace) : table(kRxWord);
        if (e == 'D' || e == 'S' || e == 'W') t = negate(t);
        r.insert(r.end(), t.begin(), t.end());
        return;
      }
      case 'b': case 'B': case '<': case '>':
        if (in_class && e == 'b') fail(kUnsupported, at, "\\b inside a class");
        fail(kUnsupported, at, "word boundaries (\\b \\B \\< \\>)");
      case 'p': case 'P': fail(kUnsupported, at, "Unicode property classes (\\p, \\P)");
      case 'A': case 'z':
        if (in_class) fail(kInvalid, at, "unrecognized escape sequence inside a class");
        break;
      default: break;
    }
    if (e >= '0' && e <= '9') fail(kInvalid, at, "backreferences are not supported");
    if ((e >= 'a' && e <= 'z') || (e >= 'A' && e <= 'Z')) fail(kInvalid, at, "unrecognized escape sequence");
    one(e);   // escaped ASCII punctuation (or space) stands for itself
  }

  // \xHH / \uHHHH / \UHHHHHHHH, or the braced form of any of them
  uint32_t hex(size_t at, int digits) {
    auto hv = [](uint32_t c) -> int {
      if (c >= '0' && c <= '9') return int(c - '0');
      if (c >= 'a' && c <= 'f') return int(c - 'a' + 10);
      if (c >= 'A' && c <= 'F') return int(c - 'A' + 10);
      return -1;
    };
    uint64_t v = 0;
    if (!eof() && peek() == '{') {
      pos_++;
      int k = 0;
      while (!eof() && peek() != '}') {
        const int h = hv(peek());
        if (h < 0 || ++k > 8) fail(kInvalid, at, "invalid hexadecimal escape");
        v = v * 16 + uint64_t(h);
        pos_++;
      }
      if (eof()) fail(kInvalid, at, "unclosed hexadecimal escape");
      pos_++;
      if (k == 0) fail(kInvalid, at, "empty hexadecimal escape");
    } else {
      for (int k = 0; k < digits; k++) {
        if (eof() || hv(peek()) < 0) fail(kInvalid, at, "invalid hexadecimal escape");
        v = v * 16 + uint64_t(hv(peek()));
        pos_++;
      }
    }
    if (v > kMaxCp || (v >= 0xD800 && v <= 0xDFFF)) fail(kInvalid, at, "escape is not a Unicode scalar value");
    return uint32_t(v);
  }

  Ranges bracket(const Flags& f, size_t at) {
    bool neg = false;
    if (!eof() && peek() == '^') { neg = true; pos_++; }
    Ranges r;
    bool first = true;
    for (;;) {
      if (eof()) fail(kInvalid, at, "unclosed character class");
      const size_t it = pos_;
      const uint32_t c = peek();
      if (c == ']' && !first) { pos_++; break; }
      first = false;
      if (c == '[') fail(kUnsupported, it, pos_ + 1 < n_ && p_[pos_ + 1] == ':' ? "POSIX classes [[:name:]]" : "nested classes");
      if (pos_ + 1 < n_ && ((c == '&' && p_[pos_ + 1] == '&') || (c == '-' && p_[pos_ + 1] == '-') || (c == '~' && p_[pos_ + 1] == '~')))
        fail(kUnsupported, it, "class set operations (&& -- ~~)");
      bool single;
      const uint32_t lo = class_item(r, single);
      if (!single) continue;
      // a range `lo-hi`; a '-' before ']' is a literal
      if (pos_ + 1 < n_ && peek() == '-' && p_[pos_ + 1] == '-') fail(kUnsupported, pos_, "class set operations (&& -- ~~)");
      if (pos_ + 1 < n_ && peek() == '-' && p_[pos_ + 1] != ']') {
        pos_++;
        const size_t hat = pos_;
        bool s2;
        Ranges tmp;
        const uint32_t hi = class_item(tmp, s2);
        if (!s2) fail(kInvalid, hat, "invalid range boundary: a class");
        if (hi < lo) fail(kInvalid, it, "invalid range: start > end");
        r.push_back({lo, hi});
      } else {
        r.push_back({lo, lo});
      }
    }
    if (f.i) case_fold(r);
    else norm(r);
    return neg ? negate(r) : r;
  }
  // one item of a class: a single code point (returned, single = true) or a Perl class (appended to r)
  uint32_t class_item(Ranges& r, bool& single) {
    const size_t at = pos_;
    if (eof()) fail(kInvalid, at, "unclosed character class");
    if (peek() == '\\') {
      pos_++;
      if (eof()) fail(kInvalid, at, "incomplete escape sequence");
      Ranges t;
      const uint32_t e = peek();
      escape(at, t, true);
      single = !(e == 'd' || e == 'D' || e == 's' || e == 'S' || e == 'w' || e == 'W');
      if (single) return t[0].first;
      r.insert(r.end(), t.begin(), t.end());
      return 0;
    }
    single = true;
    return cp();
  }

  P group(Flags& f, uint32_t depth) {
    const size_t at = pos_;
    pos_++;   // '('
    Flags inner = f;
    if (!eof() && peek() == '?') {
      pos_++;
      if (eof()) fail(kInvalid, at, "unclosed group");
      const uint32_t c = peek();
      if (c == '=' || c == '!') fail(kInvalid, at, "look-around is not supported");
      if (c == '<' && pos_ + 1 < n_ && (p_[pos_ + 1] == '=' || p_[pos_ + 1] == '!')) fail(kInvalid, at, "look-around is not supported");
      if (c == 'P' || c == '<') {
        if (c == 'P') {
          pos_++;
          if (eof() || peek() != '<') fail(kInvalid, at, "invalid capture group name syntax");
        }
        pos_++;
        capture_name(at);
      } else {
        // flags: (?flags) or (?flags:...)
        Flags g = f;
        bool negate_on = false, any = false, dangling = false;
        std::string seen;
        for (;;) {
          if (eof()) fail(kInvalid, at, "unclosed group");
          const uint32_t fc = peek();
          if (fc == ')' || fc == ':') break;
          pos_++;
          if (fc == '-') {
            if (negate_on) fail(kInvalid, at, "repeated flag negation");
            negate_on = true;
            dangling = true;
            continue;
          }
          if (seen.find(char(fc)) != std::string::npos) fail(kInvalid, at, "duplicate flag");
          if (fc < 0x80) seen.push_back(char(fc));
          dangling = false;
          any = true;
          const bool v = !negate_on;
          switch (fc) {
            case 'i': g.i = v; break;
            case 'm': g.m = v; break;
            case 's': g.s = v; break;
            case 'U': break;   // swap greed: the same match test
            case 'u': if (!v) fail(kUnsupported, at, "the flag -u"); break;
            case 'x': case 'R': fail(kUnsupported, at, std::string("the flag ") + char(fc));
            default: fail(kInvalid, at, "unrecognized flag");
          }
        }
        if (dangling) fail(kInvalid, at, "dangling flag negation");
        if (!any && !negate_on && peek() == ')') fail(kInvalid, at, "empty flag group");   // (?:...) is a plain group
        if (peek() == ')') {
          pos_++;
          f = g;   // the rest of the enclosing group
          return nullptr;
        }
        pos_++;   // ':'
        inner = g;
      }
    }
    P body = alternation(inner, depth + 1);
    if (eof() || peek() != ')') fail(kInvalid, at, "unclosed group");
    pos_++;
    return body;
  }
  void capture_name(size_t at) {
    const size_t s = pos_;
    while (!eof() && peek() != '>') {
      const uint32_t c = peek();
      if (c >= 0x80) fail(kUnsupported, at, "non-ASCII capture group name");
      const bool ok = (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_' ||
                      (pos_ > s && ((c >= '0' && c <= '9') || c == '.' || c == '[' || c == ']'));
      if (!ok) fail(kInvalid, at, "invalid capture group name");
      pos_++;
    }
    if (eof()) fail(kInvalid, at, "unclosed capture group name");
    if (pos_ == s) fail(kInvalid, at, "empty capture group name");
    std::string name(reinterpret_cast<const char*>(p_ + s), pos_ - s);
    if (std::find(names_.begin(), names_.end(), name) != names_.end()) fail(kInvalid, at, "duplicate capture group name");
    names_.push_back(name);
    pos_++;   // '>'
  }
};

// ---- UTF-8 byte-range sequences of a code point range (Russ Cox's utf8 range splitting) ----
struct Seq {
  uint8_t n;
  uint8_t lo[4], hi[4];
};
int enc(uint32_t c, uint8_t* b) {
  if (c < 0x80) { b[0] = uint8_t(c); return 1; }
  if (c < 0x800) { b[0] = uint8_t(0xC0 | (c >> 6)); b[1] = uint8_t(0x80 | (c & 0x3F)); return 2; }
  if (c < 0x10000) { b[0] = uint8_t(0xE0 | (c >> 12)); b[1] = uint8_t(0x80 | ((c >> 6) & 0x3F)); b[2] = uint8_t(0x80 | (c & 0x3F)); return 3; }
  b[0] = uint8_t(0xF0 | (c >> 18)); b[1] = uint8_t(0x80 | ((c >> 12) & 0x3F)); b[2] = uint8_t(0x80 | ((c >> 6) & 0x3F));
  b[3] = uint8_t(0x80 | (c & 0x3F));
  return 4;
}
void utf8_seqs(uint32_t lo, uint32_t hi, std::vector<Seq>& out) {
  if (lo > hi) return;
  if (lo <= 0xDFFF && hi >= 0xD800) {   // surrogates are no scalar values
    if (lo < 0xD800) utf8_seqs(lo, 0xD7FF, out);
    if (hi > 0xDFFF) utf8_seqs(0xE000, hi, out);
    return;
  }
  for (uint32_t b : {0x7Fu, 0x7FFu, 0xFFFFu}) {
    if (lo <= b && hi > b) {
      utf8_seqs(lo, b, out);
      utf8_seqs(b + 1, hi, out);
      return;
    }
  }
  if (hi < 0x80) {
    Seq s{1, {uint8_t(lo)}, {uint8_t(hi)}};
    out.push_back(s);
    return;
  }
  for (int i = 1; i < 4; i++) {
    const uint32_t m = (1u << (6 * i)) - 1;
    if ((lo & ~m) != (hi & ~m)) {
      if ((lo & m) != 0) { utf8_seqs(lo, lo | m, out); utf8_seqs((lo | m) + 1, hi, out); return; }
      if ((hi & m) != m) { utf8_seqs(lo, (hi & ~m) - 1, out); utf8_seqs(hi & ~m, hi, out); return; }
    }
  }
  Seq s{};
  uint8_t a[4], b[4];
  s.n = uint8_t(enc(lo, a));
  enc(hi, b);
  for (int k = 0; k < s.n; k++) { s.lo[k] = a[k]; s.hi[k] = b[k]; }
  out.push_back(s);
}

// ---- Thompson NFA over bytes ----
enum StKind : uint8_t { S_RANGE, S_SPLIT, S_EPS, S_ASSERT, S_MATCH, S_FAIL };
struct St {
  StKind kind;
  uint8_t lo = 0, hi = 0;
  uint32_t akind = 0;
  int32_t out = -1, out1 = -1;
};
struct Frag {
  int32_t start, end;   // `end` is an S_EPS whose `out` is patched by the caller
};

class Nfa {
 public:
  std::vector<St> st;

  int32_t add(St s) {
    if (st.size() >= kRxMaxNfa) too_large("more than 65536 NFA states");
    st.push_back(s);
    return int32_t(st.size() - 1);
  }
  int32_t eps() { return add(St{S_EPS}); }

  Frag build(const Node& n) {
    switch (n.kind) {
      case N_EMPTY: { const int32_t e = eps(); return {e, e}; }
      case N_ASSERT: {
        const int32_t e = eps();
        St a{S_ASSERT};
        a.akind = n.akind;
        a.out = e;
        return {add(a), e};
      }
      case N_SET: return set(n.set);
      case N_CONCAT: {
        Frag f = build(*n.kids[0]);
        for (size_t i = 1; i < n.kids.size(); i++) {
          const Frag g = build(*n.kids[i]);
          st[f.end].out = g.start;
          f.end = g.end;
        }
        return f;
      }
      case N_ALT: {
        const int32_t e = eps();
        int32_t start = -1, prev_split = -1;
        for (size_t i = 0; i < n.kids.size(); i++) {
          const Frag g = build(*n.kids[i]);
          st[g.end].out = e;
          if (i + 1 == n.kids.size()) {
            if (prev_split < 0) start = g.start;
            else st[prev_split].out1 = g.start;
          } else {
            St s{S_SPLIT};
            s.out = g.start;
            const int32_t si = add(s);
            if (prev_split < 0) start = si;
            else st[prev_split].out1 = si;
            prev_split = si;
          }
        }
        return {start, e};
      }
      case N_REPEAT: {
        const Node& k = *n.kids[0];
        const int32_t start = eps();
        Frag f{start, start};
        for (uint32_t i = 0; i < n.min; i++) {
          const Frag g = build(k);
          st[f.end].out = g.start;
          f.end = g.end;
        }
        const int32_t e = eps();
        if (n.max == ~0u) {
          const Frag g = build(k);
          St s{S_SPLIT};
          s.out = g.start;
          s.out1 = e;
          const int32_t si = add(s);
          st[g.end].out = si;
          st[f.end].out = si;
        } else {
          for (uint32_t i = n.min; i < n.max; i++) {
            const Frag g = build(k);
            St s{S_SPLIT};
            s.out = g.start;
            s.out1 = e;
            const int32_t si = add(s);
            st[f.end].out = si;
            f.end = g.end;
          }
          st[f.end].out = e;
        }
        return {start, e};
      }
    }
    return {-1, -1};
  }

 private:
  Frag set(const Ranges& r) {
    const int32_t e = eps();
    std::vector<Seq> seqs;
    for (auto& x : r) utf8_seqs(x.first, x.second, seqs);
    if (seqs.empty()) return {add(St{S_FAIL}), e};
    // suffix sharing: (lo, hi, next) -> state
    std::map<std::tuple<uint8_t, uint8_t, int32_t>, int32_t> cache;
    auto range = [&](uint8_t lo, uint8_t hi, int32_t next) {
      auto key = std::make_tuple(lo, hi, next);
      auto it = cache.find(key);
      if (it != cache.end()) return it->second;
      St s{S_RANGE};
      s.lo = lo;
      s.hi = hi;
      s.out = next;
      const int32_t id = add(s);
      cache.emplace(key, id);
      return id;
    };
    std::vector<int32_t> leads;
    for (const Seq& q : seqs) {
      int32_t t = e;
      for (int k = q.n - 1; k >= 0; k--) t = range(q.lo[k], q.hi[k], t);
      if (std::find(leads.begin(), leads.end(), t) == leads.end()) leads.push_back(t);
    }
    int32_t start = leads.back();
    for (size_t i = leads.size() - 1; i-- > 0;) {
      St s{S_SPLIT};
      s.out = leads[i];
      s.out1 = start;
      start = add(s);
    }
    return {start, e};
  }
};

// ---- subset construction ----
class Dfa {
 public:
  Dfa(const Nfa& nfa, int32_t start) : st_(nfa.st), mark_(nfa.st.size(), 0), start_(start) {}

  void build(std::vector<uint8_t>& blob) {
    classes();
    states_.push_back({});   // dead
    states_.push_back({});   // matched
    {
      Key k;
      k.lb = kLbStart;
      if (partial({start_}, k.lb, k.set)) start_state_ = kRxMatched;
      else start_state_ = intern(k);
    }
    std::vector<uint16_t> next;
    std::vector<uint8_t> eot;
    for (uint32_t d = 0; d < states_.size(); d++) {
      if (size_t(states_.size()) * ncls_ * 2 > kRxMaxTable) too_large("transition table over 1 MiB");
      next.resize(size_t(d + 1) * ncls_, 0);
      eot.resize(d / 8 + 1, 0);
      if (d == kRxDead) continue;
      if (d == kRxMatched) {
        for (uint32_t c = 0; c < ncls_; c++) next[size_t(d) * ncls_ + c] = kRxMatched;
        eot[d / 8] |= uint8_t(1u << (d % 8));
        continue;
      }
      const Key k = states_[d];   // copy: intern() grows states_
      std::vector<int32_t> cl;
      if (full(k, kLaEot, cl)) eot[d / 8] |= uint8_t(1u << (d % 8));
      for (int nl = 0; nl < 2; nl++) {
        const bool matched = full(k, nl ? kLaNl : 0u, cl);
        for (uint32_t c = 0; c < ncls_; c++) {
          if ((rep_[c] == '\n') != (nl == 1)) continue;
          uint32_t to = kRxMatched;
          if (!matched) {
            Key seeds;   // the NFA states after the byte, and the look-behind it leaves
            seeds.lb = nl ? kLbNl : 0u;
            for (int32_t s : cl)
              if (st_[s].kind == S_RANGE && rep_[c] >= st_[s].lo && rep_[c] <= st_[s].hi) seeds.set.push_back(st_[s].out);
            std::sort(seeds.set.begin(), seeds.set.end());
            auto it = step_.find(seeds);   // many classes reach the same seeds (the `.*?` loop alone, for one)
            if (it != step_.end()) to = it->second;
            else {
              Key nk;
              nk.lb = seeds.lb;
              to = partial(seeds.set, nk.lb, nk.set) ? kRxMatched : (nk.set.empty() ? kRxDead : intern(nk));
              work_ += seeds.set.size();
              step_.emplace(std::move(seeds), to);
            }
          }
          next[size_t(d) * ncls_ + c] = uint16_t(to);
        }
      }
    }
    const uint32_t ns = uint32_t(states_.size());
    const size_t bytes = kRxNextOff + size_t(ns) * ncls_ * 2 + (ns + 7) / 8;
    blob.assign(bytes, 0);
    RxHeader h{ns, ncls_, start_state_, uint32_t(bytes)};
    std::memcpy(blob.data(), &h, sizeof h);
    std::memcpy(blob.data() + kRxClsOff, cls_, 256);
    std::memcpy(blob.data() + kRxNextOff, next.data(), size_t(ns) * ncls_ * 2);
    std::memcpy(blob.data() + kRxNextOff + size_t(ns) * ncls_ * 2, eot.data(), (ns + 7) / 8);
  }

 private:
  static constexpr uint32_t kLbStart = 1, kLbNl = 2;   // look-behind: start of text / previous byte '\n'
  static constexpr uint32_t kLaEot = 1, kLaNl = 2;     // look-ahead: end of text / next byte '\n'
  static constexpr uint64_t kMaxWork = 1ull << 27;     // closure visits and stored set entries

  struct Key {
    uint32_t lb = 0;
    std::vector<int32_t> set;   // sorted: S_RANGE states and unresolved look-ahead assertions
    bool operator<(const Key& o) const { return lb != o.lb ? lb < o.lb : set < o.set; }
  };
  const std::vector<St>& st_;
  std::vector<uint32_t> mark_;
  uint32_t gen_ = 0;
  int32_t start_;
  uint32_t start_state_ = 0;
  uint8_t cls_[256];
  uint32_t ncls_ = 0;
  std::vector<uint32_t> rep_;   // a byte of each class
  std::vector<Key> states_;
  std::map<Key, uint32_t> index_;
  std::map<Key, uint32_t> step_;   // seeds after a byte -> DFA state
  uint64_t work_ = 0;

  void classes() {
    bool cut[257] = {};
    cut[0] = cut['\n'] = cut['\n' + 1] = true;
    for (const St& s : st_)
      if (s.kind == S_RANGE) { cut[s.lo] = true; cut[s.hi + 1] = true; }
    for (int b = 0; b < 256; b++) {
      if (cut[b]) { rep_.push_back(uint32_t(b)); ncls_++; }
      cls_[b] = uint8_t(ncls_ - 1);
    }
  }

  uint32_t intern(Key& k) {
    if (k.lb && !std::any_of(k.set.begin(), k.set.end(), [&](int32_t s) { return st_[s].kind == S_ASSERT; }))
      k.lb = 0;   // nothing left that looks behind later
    auto it = index_.find(k);
    if (it != index_.end()) return it->second;
    if (states_.size() >= kRxMaxDfa) too_large("more than 4096 DFA states");
    work_ += k.set.size();
    if (work_ > kMaxWork) too_large("subset construction over its work bound");
    const uint32_t id = uint32_t(states_.size());
    states_.push_back(k);
    index_.emplace(k, id);
    return id;
  }

  // epsilon closure from `seeds`.  la_known: resolve look-aheads with `la`; otherwise keep them as members.
  // Returns whether S_MATCH was reached; `out` gets the S_RANGE members (and unresolved look-aheads), sorted.
  bool closure(const std::vector<int32_t>& seeds, uint32_t lb, bool la_known, uint32_t la, std::vector<int32_t>& out) {
    if (++gen_ == 0) { std::fill(mark_.begin(), mark_.end(), 0); gen_ = 1; }
    out.clear();
    std::vector<int32_t> stack(seeds.rbegin(), seeds.rend());
    bool match = false;
    while (!stack.empty()) {
      const int32_t s = stack.back();
      stack.pop_back();
      if (s < 0 || mark_[s] == gen_) continue;
      mark_[s] = gen_;
      if (++work_ > kMaxWork) too_large("subset construction over its work bound");
      const St& x = st_[s];
      switch (x.kind) {
        case S_RANGE: out.push_back(s); break;
        case S_MATCH: match = true; break;
        case S_FAIL: break;
        case S_EPS: stack.push_back(x.out); break;
        case S_SPLIT: stack.push_back(x.out1); stack.push_back(x.out); break;
        case S_ASSERT: {
          bool pass;
          if (x.akind == A_START_TEXT) pass = lb & kLbStart;
          else if (x.akind == A_START_LINE) pass = lb != 0;
          else if (!la_known) { out.push_back(s); break; }
          else if (x.akind == A_END_TEXT) pass = la & kLaEot;
          else pass = la != 0;
          if (pass) stack.push_back(x.out);
          break;
        }
      }
    }
    std::sort(out.begin(), out.end());
    return match;
  }
  bool partial(const std::vector<int32_t>& seeds, uint32_t lb, std::vector<int32_t>& out) {
    return closure(seeds, lb, false, 0, out);
  }
  bool full(const Key& k, uint32_t la, std::vector<int32_t>& out) { return closure(k.set, k.lb, true, la, out); }
};

}  // namespace

int regex_compile(const char* pat, size_t n, bool case_insensitive, std::vector<uint8_t>& blob, std::string& err) {
  try {
    if (n > kRxMaxPattern) too_large("pattern over 64 KiB");
    const uint8_t* p = reinterpret_cast<const uint8_t*>(pat ? pat : "");
    Parser ps(p, n);
    Flags f;
    f.i = case_insensitive;
    P ast = ps.parse(f);
    Nfa nfa;
    // unanchored search: start = split(pattern, any byte -> start)
    St sp{S_SPLIT};
    const int32_t start = nfa.add(sp);
    St loop{S_RANGE};
    loop.lo = 0;
    loop.hi = 255;
    loop.out = start;
    const int32_t li = nfa.add(loop);
    const Frag body = nfa.build(*ast);
    nfa.st[body.end].out = nfa.add(St{S_MATCH});
    nfa.st[start].out = body.start;
    nfa.st[start].out1 = li;
    Dfa dfa(nfa, start);
    dfa.build(blob);
    return 0;
  } catch (const RxError& e) {
    err = e.msg;
    blob.clear();
    return e.code;
  } catch (const std::bad_alloc&) {
    err = "regular expression too large for the device DFA: out of host memory";
    blob.clear();
    return kUnsupported;
  }
}

}  // namespace pqb
