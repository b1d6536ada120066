// The names of test cases (docs/SPEC.md sections 5, 10 and 16), shared by the command line and the library: the method
// string of a header line, the case name, and step 2 of the section-16 matching of the cases of a revision pair.
#pragma once
#include <cctype>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/tosemscan.h"

namespace tsm_names {

inline bool is_w(unsigned char c) { return c == 0x20 || c == 0x09 || c == 0x0D || c == 0x0B || c == 0x0C; }

// docs/SPEC.md section 5
inline std::string method_string(int ext, const uint8_t* line, uint32_t len) {   // docs/SPEC.md section 5
  uint32_t b = 0, e = len;
  while (b < e && is_w(line[b])) ++b;
  while (e > b && is_w(line[e - 1])) --e;
  auto sw = [&](uint32_t i, const char* pat) { const size_t m = strlen(pat); return i + m <= e && memcmp(line + i, pat, m) == 0; };
  std::string o;
  if (ext == TSM_EXT_PY) {
    uint32_t i = b;
    if (sw(i, "class")) i += 5;
    while (i < e) {
      if (sw(i, "def")) { i += 3; continue; }
      if (!is_w(line[i])) o += (char)line[i];
      ++i;
    }
    if (!o.empty() && o.back() == ':') o.pop_back();
  } else if (ext == TSM_EXT_JAVA) {
    static const char* const words[] = {"public", "private", "protected", "static", "void", "class"};
    uint32_t i = b;
    while (i < e) {
      bool hit = false;
      for (const char* w : words) if (sw(i, w)) { i += (uint32_t)strlen(w); hit = true; break; }
      if (hit) continue;
      if (!is_w(line[i])) o += (char)line[i];
      ++i;
    }
  } else {
    uint32_t t = b;
    while (t < e && line[t] != ')') ++t;
    uint32_t s = b, u = t;
    while (s < t && (is_w(line[s]) || line[s] == '{')) ++s;
    while (u > s && (is_w(line[u - 1]) || line[u - 1] == '{')) --u;
    for (uint32_t i = s; i < u; ++i) if (line[i] != '{') o += (char)line[i];
  }
  return o;
}

// Case name of a header line: PY - identifier after `def`; C family - 2nd macro argument of TEST / TEST_F /
// TEST_P, `TEST_CASE(X)` for BOOST_AUTO_TEST_CASE(X); otherwise the SPEC section 5 method string.
inline std::string case_name(int ext, const uint8_t* line, uint32_t len) {
  uint32_t b = 0, e = len;
  while (b < e && is_w(line[b])) ++b;
  while (e > b && is_w(line[e - 1])) --e;
  const std::string s((const char*)line + b, e - b);
  if (ext == TSM_EXT_PY) {
    const size_t d = s.find("def");
    if (d != std::string::npos) {
      size_t i = d + 3;
      while (i < s.size() && is_w((unsigned char)s[i])) ++i;
      size_t j = i;
      while (j < s.size() && (isalnum((unsigned char)s[j]) || s[j] == '_')) ++j;
      if (j > i) return s.substr(i, j - i);
    }
  } else {
    auto trim = [](std::string t) { size_t a = 0, z = t.size(); while (a < z && is_w((unsigned char)t[a])) ++a; while (z > a && is_w((unsigned char)t[z - 1])) --z; return t.substr(a, z - a); };
    if (s.rfind("TEST(", 0) == 0 || s.rfind("TEST_F(", 0) == 0 || s.rfind("TEST_P(", 0) == 0) {
      const size_t c = s.find(','), r = s.find(')');
      if (c != std::string::npos && (r == std::string::npos || c < r)) return trim(s.substr(c + 1, (r == std::string::npos ? s.size() : r) - c - 1));
    }
    if (s.rfind("BOOST_AUTO_TEST_CASE(", 0) == 0) {
      const size_t r = s.find(')');
      return "TEST_CASE(" + trim(s.substr(21, (r == std::string::npos ? s.size() : r) - 21)) + ")";
    }
  }
  return method_string(ext, line, len);
}

// Step 2 of the section-16 matching: a new case j that step 1 left unmatched (match[j] < 0) is matched with the old case k
// whose name is its name when that name is held by exactly one unmatched case on each side.  na / nb: the names of the old /
// new cases; used[k]: old case k is matched (updated).
inline void match_by_name(const std::vector<std::string>& na, const std::vector<std::string>& nb, std::vector<int64_t>& match,
                          std::vector<char>& used) {
  std::map<std::string, int64_t> cnt_new, cnt_old, old_of;
  for (size_t j = 0; j < nb.size(); ++j) if (match[j] < 0) ++cnt_new[nb[j]];
  for (size_t k = 0; k < na.size(); ++k) if (!used[k]) { ++cnt_old[na[k]]; old_of[na[k]] = (int64_t)k; }
  for (size_t j = 0; j < nb.size(); ++j)
    if (match[j] < 0 && cnt_new[nb[j]] == 1 && cnt_old[nb[j]] == 1) { match[j] = old_of[nb[j]]; used[(size_t)match[j]] = 1; }
}

}  // namespace tsm_names
