// TEST INFRASTRUCTURE ONLY.  Minimal stand-in for the subset of abseil-cpp (pinned by the reference at tag
// 20250814.1, open_spiel/scripts/global_variables.sh:33; not vendored) that the reference
// files on the hot path include.  It lets oracle/ref_build.mk compile those reference sources UNMODIFIED,
// from the OpenSpiel checkout, into oracle/_ref/.  Everything maps onto the C++20 standard library.
// Written from the documented abseil API; no abseil source was available or copied.
//
// RNG note: absl::uniform_int_distribution / absl::Uniform(int) below restate abseil's published algorithm
// (FastUniformBits word assembly, power-of-two mask fast path, Lemire multiply-shift with rejection) from
// its documentation; absl::Uniform(double) is a plain 53-bit mantissa draw.  No reference test pins values
// at this boundary (SURVEY.md §8c), so seeded-stream parity with stock OpenSpiel binaries is UNPINNED.
#ifndef B2S_ABSL_SHIM_ALL_H_
#define B2S_ABSL_SHIM_ALL_H_

#include <algorithm>
#include <charconv>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>
#include <optional>
#include <random>
#include <set>
#include <string>
#include <string_view>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#define ABSL_GUARDED_BY(x)
#define ABSL_PT_GUARDED_BY(x)
#define ABSL_EXCLUSIVE_LOCKS_REQUIRED(...)
#define ABSL_LOCKS_EXCLUDED(...)
#define ABSL_DEPRECATED(msg) [[deprecated(msg)]]
#define ABSL_MUST_USE_RESULT [[nodiscard]]
#define ABSL_ATTRIBUTE_UNUSED __attribute__((unused))
#define ABSL_ATTRIBUTE_NOINLINE __attribute__((noinline))
#define ABSL_ATTRIBUTE_ALWAYS_INLINE __attribute__((always_inline))
#define ABSL_FALLTHROUGH_INTENDED [[fallthrough]]

namespace absl {

// ---- types ------------------------------------------------------------------------------------------
using string_view = std::string_view;
template <typename T> using optional = std::optional<T>;
using nullopt_t = std::nullopt_t;
inline constexpr std::nullopt_t nullopt = std::nullopt;
using std::make_optional;
using std::make_unique;

template <typename T>
class Span {
 public:
  using value_type = std::remove_cv_t<T>;
  using iterator = T*;
  using const_iterator = const T*;
  using size_type = size_t;
  constexpr Span() : p_(nullptr), n_(0) {}
  constexpr Span(T* p, size_t n) : p_(p), n_(n) {}
  template <size_t N> constexpr Span(T (&a)[N]) : p_(a), n_(N) {}
  template <typename V, typename = std::enable_if_t<
                            !std::is_same_v<std::decay_t<V>, Span> &&
                            std::is_convertible_v<decltype(std::declval<V&>().data()), T*>>>
  constexpr Span(V& v) : p_(v.data()), n_(v.size()) {}
  template <typename V, typename = std::enable_if_t<
                            std::is_const_v<T> && !std::is_same_v<std::decay_t<V>, Span> &&
                            std::is_convertible_v<decltype(std::declval<const V&>().data()), T*>>, int = 0>
  constexpr Span(const V& v) : p_(v.data()), n_(v.size()) {}
  template <typename U = T, typename = std::enable_if_t<std::is_const_v<U>>>
  Span(std::initializer_list<value_type> l) : p_(l.begin()), n_(l.size()) {}
  constexpr T* data() const { return p_; }
  constexpr size_t size() const { return n_; }
  constexpr size_t length() const { return n_; }
  constexpr bool empty() const { return n_ == 0; }
  constexpr T& operator[](size_t i) const { return p_[i]; }
  constexpr T& at(size_t i) const { return p_[i]; }
  constexpr T& front() const { return p_[0]; }
  constexpr T& back() const { return p_[n_ - 1]; }
  constexpr T* begin() const { return p_; }
  constexpr T* end() const { return p_ + n_; }
  constexpr Span subspan(size_t pos = 0, size_t len = static_cast<size_t>(-1)) const {
    return Span(p_ + pos, std::min(len, n_ - pos));
  }
  constexpr Span first(size_t n) const { return Span(p_, n); }
  constexpr Span last(size_t n) const { return Span(p_ + n_ - n, n); }
 private:
  T* p_;
  size_t n_;
};
template <typename T> constexpr Span<T> MakeSpan(T* p, size_t n) { return Span<T>(p, n); }
template <typename T> constexpr Span<T> MakeSpan(T* b, T* e) { return Span<T>(b, e - b); }
template <typename C> constexpr auto MakeSpan(C& c) { return Span<std::remove_pointer_t<decltype(c.data())>>(c.data(), c.size()); }
template <typename T, size_t N> constexpr Span<T> MakeSpan(T (&a)[N]) { return Span<T>(a, N); }
template <typename T> constexpr Span<const T> MakeConstSpan(const T* p, size_t n) { return Span<const T>(p, n); }
template <typename C> constexpr auto MakeConstSpan(const C& c) { return Span<const std::remove_pointer_t<decltype(c.data())>>(c.data(), c.size()); }

// ---- containers ---------------------------------------------------------------------------------------
template <typename K, typename V, typename H = std::hash<K>, typename E = std::equal_to<K>>
using flat_hash_map = std::unordered_map<K, V, H, E>;
template <typename K, typename V, typename H = std::hash<K>, typename E = std::equal_to<K>>
using node_hash_map = std::unordered_map<K, V, H, E>;
template <typename K, typename H = std::hash<K>, typename E = std::equal_to<K>>
using flat_hash_set = std::unordered_set<K, H, E>;
template <typename K, typename V, typename C = std::less<K>> using btree_map = std::map<K, V, C>;
template <typename K, typename C = std::less<K>> using btree_set = std::set<K, C>;
template <typename T, size_t N, typename A = std::allocator<T>> using InlinedVector = std::vector<T, A>;

// ---- algorithm/container.h ------------------------------------------------------------------------------
template <typename C, typename T> auto c_find(C& c, const T& v) { return std::find(std::begin(c), std::end(c), v); }
template <typename C, typename P> auto c_find_if(C& c, P p) { return std::find_if(std::begin(c), std::end(c), p); }
template <typename C, typename T> bool c_linear_search(const C& c, const T& v) { return std::find(std::begin(c), std::end(c), v) != std::end(c); }
template <typename C, typename F> F c_for_each(C&& c, F f) { return std::for_each(std::begin(c), std::end(c), f); }
template <typename C, typename T> void c_fill(C& c, const T& v) { std::fill(std::begin(c), std::end(c), v); }
template <typename C, typename T> void c_iota(C& c, const T& v) { std::iota(std::begin(c), std::end(c), v); }
template <typename C, typename P> bool c_all_of(const C& c, P p) { return std::all_of(std::begin(c), std::end(c), p); }
template <typename C, typename P> bool c_any_of(const C& c, P p) { return std::any_of(std::begin(c), std::end(c), p); }
template <typename C, typename T> T c_accumulate(const C& c, T init) { return std::accumulate(std::begin(c), std::end(c), std::move(init)); }
template <typename C, typename T, typename F> T c_accumulate(const C& c, T init, F f) { return std::accumulate(std::begin(c), std::end(c), std::move(init), f); }
template <typename C> void c_sort(C& c) { std::sort(std::begin(c), std::end(c)); }
template <typename C, typename F> void c_sort(C& c, F f) { std::sort(std::begin(c), std::end(c), f); }
template <typename C> auto c_max_element(C& c) { return std::max_element(std::begin(c), std::end(c)); }
template <typename C> auto c_min_element(C& c) { return std::min_element(std::begin(c), std::end(c)); }
template <typename C, typename T> auto c_count(const C& c, const T& v) { return std::count(std::begin(c), std::end(c), v); }
template <typename C, typename P> auto c_count_if(const C& c, P p) { return std::count_if(std::begin(c), std::end(c), p); }
template <typename C> void c_reverse(C& c) { std::reverse(std::begin(c), std::end(c)); }

// ---- strings: AlphaNum / StrCat / StrAppend ---------------------------------------------------------------
namespace shim_internal {
inline std::string SixDigits(double d) {     // StrCat(double): "%g" with six significant digits
  char b[64];
  snprintf(b, sizeof b, "%g", d);
  return b;
}
}  // namespace shim_internal

class AlphaNum {
 public:
  AlphaNum(int v) : s_(std::to_string(v)) {}
  AlphaNum(unsigned v) : s_(std::to_string(v)) {}
  AlphaNum(long v) : s_(std::to_string(v)) {}
  AlphaNum(unsigned long v) : s_(std::to_string(v)) {}
  AlphaNum(long long v) : s_(std::to_string(v)) {}
  AlphaNum(unsigned long long v) : s_(std::to_string(v)) {}
  AlphaNum(short v) : s_(std::to_string(v)) {}
  AlphaNum(unsigned short v) : s_(std::to_string(v)) {}
  AlphaNum(signed char v) : s_(std::to_string((int)v)) {}
  AlphaNum(unsigned char v) : s_(std::to_string((int)v)) {}
  AlphaNum(bool v) : s_(v ? "1" : "0") {}
  AlphaNum(float v) : s_(shim_internal::SixDigits(v)) {}
  AlphaNum(double v) : s_(shim_internal::SixDigits(v)) {}
  AlphaNum(const char* v) : s_(v ? v : "") {}
  AlphaNum(const std::string& v) : s_(v) {}
  AlphaNum(std::string_view v) : s_(v) {}
  AlphaNum(char) = delete;
  template <typename E, typename = std::enable_if_t<std::is_enum_v<E>>>
  AlphaNum(E e) : s_(std::to_string(static_cast<long long>(static_cast<std::underlying_type_t<E>>(e)))) {}
  const std::string& str() const { return s_; }
 private:
  std::string s_;
};

inline std::string StrCat() { return std::string(); }
template <typename... A>
std::string StrCat(const A&... a) {
  std::string out;
  ((out += AlphaNum(a).str()), ...);
  return out;
}
template <typename... A>
void StrAppend(std::string* dest, const A&... a) {
  ((*dest += AlphaNum(a).str()), ...);
}

// ---- strings: StrFormat ------------------------------------------------------------------------------------
namespace shim_internal {
struct FormatArg {
  enum Kind { kInt, kUint, kDouble, kString, kChar, kPtr } kind;
  long long i = 0;
  unsigned long long u = 0;
  double d = 0;
  std::string s;
  const void* p = nullptr;
  FormatArg(bool v) : kind(kInt), i(v) {}
  FormatArg(char v) : kind(kChar), i(v) {}
  FormatArg(signed char v) : kind(kInt), i(v) {}
  FormatArg(unsigned char v) : kind(kUint), u(v) {}
  FormatArg(short v) : kind(kInt), i(v) {}
  FormatArg(unsigned short v) : kind(kUint), u(v) {}
  FormatArg(int v) : kind(kInt), i(v) {}
  FormatArg(unsigned v) : kind(kUint), u(v) {}
  FormatArg(long v) : kind(kInt), i(v) {}
  FormatArg(unsigned long v) : kind(kUint), u(v) {}
  FormatArg(long long v) : kind(kInt), i(v) {}
  FormatArg(unsigned long long v) : kind(kUint), u(v) {}
  FormatArg(float v) : kind(kDouble), d(v) {}
  FormatArg(double v) : kind(kDouble), d(v) {}
  FormatArg(long double v) : kind(kDouble), d((double)v) {}
  FormatArg(const char* v) : kind(kString), s(v ? v : "(null)") {}
  FormatArg(const std::string& v) : kind(kString), s(v) {}
  FormatArg(std::string_view v) : kind(kString), s(v) {}
  template <typename E, typename = std::enable_if_t<std::is_enum_v<E>>>
  FormatArg(E e) : kind(kInt), i(static_cast<long long>(static_cast<std::underlying_type_t<E>>(e))) {}
  template <typename T> FormatArg(T* v) : kind(kPtr), p(v) {}
  long long as_int() const { return kind == kUint ? (long long)u : kind == kDouble ? (long long)d : i; }
  unsigned long long as_uint() const { return kind == kUint ? u : kind == kDouble ? (unsigned long long)d : (unsigned long long)i; }
  double as_double() const { return kind == kDouble ? d : kind == kUint ? (double)u : (double)i; }
};

inline std::string FormatImpl(std::string_view fmt, const std::vector<FormatArg>& args) {
  std::string out;
  size_t ai = 0;
  for (size_t k = 0; k < fmt.size(); ++k) {
    char c = fmt[k];
    if (c != '%') { out += c; continue; }
    if (k + 1 < fmt.size() && fmt[k + 1] == '%') { out += '%'; ++k; continue; }
    std::string spec = "%";
    ++k;
    while (k < fmt.size() && strchr("-+ #0", fmt[k])) spec += fmt[k++];
    auto take_star = [&]() { int v = ai < args.size() ? (int)args[ai].as_int() : 0; ++ai; return std::to_string(v); };
    if (k < fmt.size() && fmt[k] == '*') { spec += take_star(); ++k; }
    while (k < fmt.size() && isdigit((unsigned char)fmt[k])) spec += fmt[k++];
    if (k < fmt.size() && fmt[k] == '.') {
      spec += fmt[k++];
      if (k < fmt.size() && fmt[k] == '*') { spec += take_star(); ++k; }
      while (k < fmt.size() && isdigit((unsigned char)fmt[k])) spec += fmt[k++];
    }
    while (k < fmt.size() && strchr("hlLqjzt", fmt[k])) ++k;      // length modifiers are ignored
    if (k >= fmt.size()) break;
    char conv = fmt[k];
    if (ai >= args.size()) { out += "<missing arg>"; continue; }
    const FormatArg& a = args[ai++];
    char buf[512];
    if (conv == 'v') conv = a.kind == FormatArg::kString ? 's' : a.kind == FormatArg::kDouble ? 'g'
                          : a.kind == FormatArg::kUint ? 'u' : a.kind == FormatArg::kChar ? 'c' : 'd';
    switch (conv) {
      case 'd': case 'i':
        snprintf(buf, sizeof buf, (spec + "lld").c_str(), a.as_int()); out += buf; break;
      case 'u': case 'x': case 'X': case 'o':
        snprintf(buf, sizeof buf, (spec + "ll" + conv).c_str(), a.as_uint()); out += buf; break;
      case 'f': case 'F': case 'e': case 'E': case 'g': case 'G': case 'a': case 'A':
        snprintf(buf, sizeof buf, (spec + conv).c_str(), a.as_double()); out += buf; break;
      case 'c':
        snprintf(buf, sizeof buf, (spec + "c").c_str(), (int)a.as_int()); out += buf; break;
      case 's': {
        std::string v = a.kind == FormatArg::kString ? a.s
                        : a.kind == FormatArg::kDouble ? SixDigits(a.d)
                        : a.kind == FormatArg::kUint ? std::to_string(a.u) : std::to_string(a.i);
        int n = snprintf(nullptr, 0, (spec + "s").c_str(), v.c_str());
        std::string tmp(n + 1, '\0');
        snprintf(tmp.data(), n + 1, (spec + "s").c_str(), v.c_str());
        tmp.resize(n);
        out += tmp;
        break;
      }
      case 'p':
        snprintf(buf, sizeof buf, "%p", a.p); out += buf; break;
      default:
        out += spec; out += conv;
    }
  }
  return out;
}
}  // namespace shim_internal

template <typename... A>
std::string StrFormat(std::string_view fmt, const A&... a) {
  return shim_internal::FormatImpl(fmt, std::vector<shim_internal::FormatArg>{shim_internal::FormatArg(a)...});
}
template <typename... A>
std::string StreamFormat(std::string_view fmt, const A&... a) { return StrFormat(fmt, a...); }
template <typename... A>
void StrAppendFormat(std::string* dst, std::string_view fmt, const A&... a) { *dst += StrFormat(fmt, a...); }

// ---- strings: StrJoin ----------------------------------------------------------------------------------------
struct AlphaNumFormatterImpl {
  template <typename T> void operator()(std::string* out, const T& v) const { StrAppend(out, v); }
};
inline AlphaNumFormatterImpl AlphaNumFormatter() { return {}; }
template <typename F1, typename F2>
struct PairFormatterImpl {
  F1 f1; std::string sep; F2 f2;
  template <typename P> void operator()(std::string* out, const P& p) const { f1(out, p.first); *out += sep; f2(out, p.second); }
};
template <typename F1, typename F2>
PairFormatterImpl<F1, F2> PairFormatter(F1 f1, std::string_view sep, F2 f2) { return {f1, std::string(sep), f2}; }
inline auto PairFormatter(std::string_view sep) { return PairFormatter(AlphaNumFormatter(), sep, AlphaNumFormatter()); }

template <typename It, typename F>
std::string StrJoin(It b, It e, std::string_view sep, F&& f) {
  std::string out;
  bool first = true;
  for (; b != e; ++b) { if (!first) out += sep; first = false; f(&out, *b); }
  return out;
}
template <typename R, typename F>
std::string StrJoin(const R& r, std::string_view sep, F&& f) { return StrJoin(std::begin(r), std::end(r), sep, f); }
template <typename R>
std::string StrJoin(const R& r, std::string_view sep) { return StrJoin(std::begin(r), std::end(r), sep, AlphaNumFormatter()); }
template <typename T>
std::string StrJoin(std::initializer_list<T> r, std::string_view sep) { return StrJoin(r.begin(), r.end(), sep, AlphaNumFormatter()); }

// ---- strings: StrSplit ----------------------------------------------------------------------------------------
struct ByChar { char c; explicit ByChar(char ch) : c(ch) {} };
struct ByString { std::string s; explicit ByString(std::string_view sv) : s(sv) {} };
namespace shim_internal {
struct Delim {
  std::string s;
  int limit = -1;
  Delim(char c) : s(1, c) {}
  Delim(const char* p) : s(p) {}
  Delim(const std::string& p) : s(p) {}
  Delim(std::string_view p) : s(p) {}
  Delim(ByChar b) : s(1, b.c) {}
  Delim(ByString b) : s(b.s) {}
};
}  // namespace shim_internal
template <typename D>
shim_internal::Delim MaxSplits(D d, int limit) { shim_internal::Delim x(d); x.limit = limit; return x; }
struct SkipEmpty {};
struct AllowEmpty {};

class Splitter {
 public:
  Splitter(std::string_view text, const shim_internal::Delim& d, bool skip_empty) { Init(text, d, skip_empty); }
  Splitter(std::string&& owned, const shim_internal::Delim& d, bool skip_empty) : owned_(std::make_shared<std::string>(std::move(owned))) {
    Init(*owned_, d, skip_empty);
  }
  auto begin() const { return parts_.begin(); }
  auto end() const { return parts_.end(); }
  template <typename C, typename = typename C::value_type, typename = decltype(std::declval<C&>().insert(std::declval<C&>().end(), std::declval<typename C::value_type>()))>
  operator C() const {
    C c;
    for (auto p : parts_) c.insert(c.end(), typename C::value_type(p));
    return c;
  }
  template <typename A, typename B>
  operator std::pair<A, B>() const {
    return std::pair<A, B>(parts_.size() > 0 ? A(parts_[0]) : A(), parts_.size() > 1 ? B(parts_[1]) : B());
  }
 private:
  void Init(std::string_view text, const shim_internal::Delim& d, bool skip_empty) {
    size_t pos = 0;
    int splits = 0;
    if (d.s.empty()) {            // empty delimiter: split into characters
      for (size_t i = 0; i < text.size(); ++i) parts_.push_back(text.substr(i, 1));
      if (text.empty()) parts_.push_back(text);
      return;
    }
    while (true) {
      size_t hit = (d.limit >= 0 && splits >= d.limit) ? std::string_view::npos : text.find(d.s, pos);
      std::string_view piece = hit == std::string_view::npos ? text.substr(pos) : text.substr(pos, hit - pos);
      if (!(skip_empty && piece.empty())) parts_.push_back(piece);
      if (hit == std::string_view::npos) break;
      pos = hit + d.s.size();
      ++splits;
    }
  }
  std::shared_ptr<std::string> owned_;
  std::vector<std::string_view> parts_;
};
template <typename D> Splitter StrSplit(std::string_view text, D d) { return Splitter(text, shim_internal::Delim(d), false); }
template <typename D> Splitter StrSplit(std::string&& text, D d) { return Splitter(std::move(text), shim_internal::Delim(d), false); }
template <typename D> Splitter StrSplit(const char* text, D d) { return Splitter(std::string_view(text), shim_internal::Delim(d), false); }
template <typename D> Splitter StrSplit(const std::string& text, D d) { return Splitter(std::string_view(text), shim_internal::Delim(d), false); }
template <typename D> Splitter StrSplit(std::string_view text, D d, SkipEmpty) { return Splitter(text, shim_internal::Delim(d), true); }

// ---- strings: misc ------------------------------------------------------------------------------------------
inline bool StrContains(std::string_view h, std::string_view n) { return h.find(n) != std::string_view::npos; }
inline bool StrContains(std::string_view h, char c) { return h.find(c) != std::string_view::npos; }
inline bool StartsWith(std::string_view s, std::string_view p) { return s.substr(0, p.size()) == p; }
inline bool EndsWith(std::string_view s, std::string_view p) { return s.size() >= p.size() && s.substr(s.size() - p.size()) == p; }
inline std::string_view StripAsciiWhitespace(std::string_view s) {
  size_t b = 0, e = s.size();
  while (b < e && isspace((unsigned char)s[b])) ++b;
  while (e > b && isspace((unsigned char)s[e - 1])) --e;
  return s.substr(b, e - b);
}
inline void StripAsciiWhitespace(std::string* s) { *s = std::string(StripAsciiWhitespace(std::string_view(*s))); }
inline std::string AsciiStrToLower(std::string_view s) { std::string r(s); for (auto& c : r) c = (char)tolower((unsigned char)c); return r; }
inline std::string AsciiStrToUpper(std::string_view s) { std::string r(s); for (auto& c : r) c = (char)toupper((unsigned char)c); return r; }
inline std::string StrReplaceAll(std::string_view s, std::initializer_list<std::pair<std::string_view, std::string_view>> reps) {
  std::string out;
  size_t i = 0;
  while (i < s.size()) {
    bool hit = false;
    for (auto& r : reps)
      if (!r.first.empty() && s.compare(i, r.first.size(), r.first) == 0) { out += r.second; i += r.first.size(); hit = true; break; }
    if (!hit) out += s[i++];
  }
  return out;
}
template <typename T>
bool SimpleAtoi(std::string_view s, T* out) {
  s = StripAsciiWhitespace(s);
  if (!s.empty() && s[0] == '+') s.remove_prefix(1);
  if (s.empty()) return false;
  T v{};
  auto r = std::from_chars(s.data(), s.data() + s.size(), v);
  if (r.ec != std::errc() || r.ptr != s.data() + s.size()) return false;
  *out = v;
  return true;
}
inline bool SimpleAtod(std::string_view s, double* out) {
  s = StripAsciiWhitespace(s);
  if (s.empty()) return false;
  std::string z(s);
  char* end = nullptr;
  double v = strtod(z.c_str(), &end);
  if (end != z.c_str() + z.size()) return false;
  *out = v;
  return true;
}
inline bool SimpleAtof(std::string_view s, float* out) { double d; if (!SimpleAtod(s, &d)) return false; *out = (float)d; return true; }
inline bool SimpleAtob(std::string_view s, bool* out) {
  std::string l = AsciiStrToLower(s);
  if (l == "true" || l == "t" || l == "yes" || l == "y" || l == "1") { *out = true; return true; }
  if (l == "false" || l == "f" || l == "no" || l == "n" || l == "0") { *out = false; return true; }
  return false;
}
enum class chars_format { scientific = 1, fixed = 2, hex = 4, general = fixed | scientific };
struct from_chars_result { const char* ptr; std::errc ec; };
inline from_chars_result from_chars(const char* first, const char* last, double& value, chars_format fmt = chars_format::general) {
  std::chars_format f = fmt == chars_format::hex ? std::chars_format::hex : fmt == chars_format::fixed ? std::chars_format::fixed
                        : fmt == chars_format::scientific ? std::chars_format::scientific : std::chars_format::general;
  // absl::from_chars parses a "0x"-prefixed number as a hex float in general mode too (that is how the reference
  // reads back its "%a" serialisation, cfr.cc:546-560); std::from_chars never accepts the prefix.
  bool neg = false;
  const char* p = first;
  const char* q = (p < last && *p == '-') ? p + 1 : p;
  const bool prefixed = last - q >= 2 && q[0] == '0' && (q[1] == 'x' || q[1] == 'X');
  if (fmt == chars_format::hex || prefixed) {
    f = std::chars_format::hex;
    if (p < last && *p == '-') { neg = true; ++p; }
    if (last - p >= 2 && p[0] == '0' && (p[1] == 'x' || p[1] == 'X')) p += 2;
    double v = 0;
    auto r = std::from_chars(p, last, v, f);
    if (r.ec == std::errc()) value = neg ? -v : v;
    return {r.ptr, r.ec};
  }
  auto r = std::from_chars(first, last, value, f);
  return {r.ptr, r.ec};
}
inline from_chars_result from_chars(const char* first, const char* last, float& value, chars_format fmt = chars_format::general) {
  double d = 0;
  auto r = from_chars(first, last, d, fmt);
  if (r.ec == std::errc()) value = (float)d;
  return r;
}

// ---- time ---------------------------------------------------------------------------------------------------
class Duration {
 public:
  constexpr Duration() : ns_(0) {}
  constexpr explicit Duration(int64_t ns) : ns_(ns) {}
  int64_t ns_;
};
class Time {
 public:
  constexpr Time() : ns_(0) {}
  constexpr explicit Time(int64_t ns) : ns_(ns) {}
  int64_t ns_;
};
inline Time Now() {
  return Time(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::system_clock::now().time_since_epoch()).count());
}
constexpr Time UnixEpoch() { return Time(0); }
inline Duration operator-(Time a, Time b) { return Duration(a.ns_ - b.ns_); }
inline Time operator+(Time a, Duration d) { return Time(a.ns_ + d.ns_); }
inline Time operator-(Time a, Duration d) { return Time(a.ns_ - d.ns_); }
inline Duration operator+(Duration a, Duration b) { return Duration(a.ns_ + b.ns_); }
inline Duration operator-(Duration a, Duration b) { return Duration(a.ns_ - b.ns_); }
inline bool operator<(Duration a, Duration b) { return a.ns_ < b.ns_; }
inline bool operator>(Duration a, Duration b) { return a.ns_ > b.ns_; }
inline bool operator<=(Duration a, Duration b) { return a.ns_ <= b.ns_; }
inline bool operator>=(Duration a, Duration b) { return a.ns_ >= b.ns_; }
inline bool operator<(Time a, Time b) { return a.ns_ < b.ns_; }
inline bool operator>(Time a, Time b) { return a.ns_ > b.ns_; }
inline double ToDoubleSeconds(Duration d) { return d.ns_ * 1e-9; }
inline double ToDoubleMilliseconds(Duration d) { return d.ns_ * 1e-6; }
inline int64_t ToInt64Nanoseconds(Duration d) { return d.ns_; }
inline int64_t ToInt64Microseconds(Duration d) { return d.ns_ / 1000; }
inline int64_t ToInt64Milliseconds(Duration d) { return d.ns_ / 1000000; }
inline int64_t ToInt64Seconds(Duration d) { return d.ns_ / 1000000000; }
inline int64_t ToUnixMicros(Time t) { return t.ns_ / 1000; }
inline int64_t ToUnixNanos(Time t) { return t.ns_; }
template <typename T> Duration Seconds(T s) { return Duration((int64_t)(s * 1e9)); }
template <typename T> Duration Milliseconds(T s) { return Duration((int64_t)(s * 1e6)); }
template <typename T> Duration Microseconds(T s) { return Duration((int64_t)(s * 1e3)); }
template <typename T> Duration Nanoseconds(T s) { return Duration((int64_t)s); }
inline Duration ZeroDuration() { return Duration(0); }
inline Duration InfiniteDuration() { return Duration(std::numeric_limits<int64_t>::max()); }

// ---- synchronization ---------------------------------------------------------------------------------------------
class Mutex {
 public:
  void Lock() { m_.lock(); }
  void Unlock() { m_.unlock(); }
 private:
  std::mutex m_;
};
class MutexLock {
 public:
  explicit MutexLock(Mutex* m) : m_(m) { m_->Lock(); }
  explicit MutexLock(Mutex& m) : m_(&m) { m_->Lock(); }
  ~MutexLock() { m_->Unlock(); }
  MutexLock(const MutexLock&) = delete;
 private:
  Mutex* m_;
};

// ---- random ------------------------------------------------------------------------------------------------------
namespace shim_internal {
// FastUniformBits<U>: assemble an unsigned word from a URBG whose range is a power of two (mt19937: 32 bits,
// mt19937_64: 64 bits); the first draw lands in the high bits.
template <typename U, typename G>
U FastBits(G& g) {
  using R = typename std::remove_reference_t<G>::result_type;
  constexpr unsigned long long lo = (std::remove_reference_t<G>::min)(), hi = (std::remove_reference_t<G>::max)();
  constexpr unsigned long long range_minus1 = hi - lo;
  constexpr int urbg_bits = range_minus1 == ~0ull ? 64 : __builtin_popcountll(range_minus1);
  static_assert((range_minus1 & (range_minus1 + 1)) == 0, "shim supports power-of-two URBG ranges only");
  constexpr int want = std::numeric_limits<U>::digits;
  constexpr int iters = (want + urbg_bits - 1) / urbg_bits;
  U r = static_cast<U>(static_cast<R>(g() - lo));
  for (int n = 1; n < iters; ++n) r = static_cast<U>(r << (urbg_bits % (8 * sizeof(U)))) + static_cast<U>(static_cast<R>(g() - lo));
  return r;
}
}  // namespace shim_internal

template <typename IntType = int>
class uniform_int_distribution {
 public:
  using result_type = IntType;
  using U = std::make_unsigned_t<IntType>;
  uniform_int_distribution() : lo_(0), range_((std::numeric_limits<U>::max)() >> (std::is_signed_v<IntType> ? 1 : 0)) {}
  explicit uniform_int_distribution(IntType lo, IntType hi = (std::numeric_limits<IntType>::max)())
      : lo_(lo), range_(static_cast<U>(hi) - static_cast<U>(lo)) {}
  template <typename G>
  result_type operator()(G& g) {
    return static_cast<result_type>(static_cast<U>(lo_) + Generate(g, range_));
  }
  result_type a() const { return lo_; }
  result_type b() const { return static_cast<result_type>(static_cast<U>(lo_) + range_); }
  result_type min() const { return a(); }
  result_type max() const { return b(); }
  void reset() {}
 private:
  template <typename G>
  static U Generate(G& g, U R) {
    U bits = shim_internal::FastBits<U>(g);
    const U Lim = R + 1;
    if ((R & Lim) == 0) return bits & R;          // power-of-two range (incl. the full range): mask
    using W = std::conditional_t<(sizeof(U) > 4), unsigned __int128, unsigned long long>;
    constexpr int N = std::numeric_limits<U>::digits;
    W product = static_cast<W>(bits) * static_cast<W>(Lim);
    if (static_cast<U>(product) < Lim) {
      const U threshold = static_cast<U>(((std::numeric_limits<U>::max)() - Lim + 1) % Lim);
      while (static_cast<U>(product) < threshold) {
        bits = shim_internal::FastBits<U>(g);
        product = static_cast<W>(bits) * static_cast<W>(Lim);
      }
    }
    return static_cast<U>(product >> N);
  }
  IntType lo_;
  U range_;
};

template <typename RealType = double>
class uniform_real_distribution {
 public:
  using result_type = RealType;
  uniform_real_distribution() : lo_(0), hi_(1) {}
  explicit uniform_real_distribution(RealType lo, RealType hi = 1) : lo_(lo), hi_(hi) {}
  template <typename G>
  result_type operator()(G& g) {
    for (;;) {
      uint64_t bits = shim_internal::FastBits<uint64_t>(g);
      RealType u = static_cast<RealType>(bits >> 11) * static_cast<RealType>(1.0 / 9007199254740992.0);
      RealType r = lo_ + u * (hi_ - lo_);
      if (r < hi_ || lo_ == hi_) return r;
    }
  }
  result_type a() const { return lo_; }
  result_type b() const { return hi_; }
  void reset() {}
 private:
  RealType lo_, hi_;
};

template <typename IntType = int>
class discrete_distribution {
 public:
  using result_type = IntType;
  discrete_distribution() {}
  template <typename It> discrete_distribution(It b, It e) : w_(b, e) {}
  discrete_distribution(std::initializer_list<double> l) : w_(l) {}
  template <typename G>
  result_type operator()(G& g) {
    double total = std::accumulate(w_.begin(), w_.end(), 0.0);
    double u = uniform_real_distribution<double>(0.0, total)(g), acc = 0;
    for (size_t i = 0; i < w_.size(); ++i) { acc += w_[i]; if (u < acc) return (IntType)i; }
    return (IntType)(w_.empty() ? 0 : w_.size() - 1);
  }
 private:
  std::vector<double> w_;
};

struct IntervalClosedClosedTag {};
struct IntervalClosedOpenTag {};
struct IntervalOpenClosedTag {};
struct IntervalOpenOpenTag {};
inline constexpr IntervalClosedClosedTag IntervalClosedClosed{};
inline constexpr IntervalClosedClosedTag IntervalClosed{};
inline constexpr IntervalClosedOpenTag IntervalClosedOpen{};
inline constexpr IntervalOpenClosedTag IntervalOpenClosed{};
inline constexpr IntervalOpenOpenTag IntervalOpenOpen{};
inline constexpr IntervalOpenOpenTag IntervalOpen{};

namespace shim_internal {
template <typename T, typename G>
T UniformImpl(G& g, T lo, T hi, bool closed_hi) {
  if constexpr (std::is_integral_v<T>) {
    if (!closed_hi) { if (!(lo < hi)) return lo; hi = hi - 1; }
    return uniform_int_distribution<T>(lo, hi)(g);
  } else {
    return uniform_real_distribution<T>(lo, hi)(g);
  }
}
}  // namespace shim_internal
template <typename R = void, typename G, typename A, typename B>
auto Uniform(G&& g, A lo, B hi) {
  using T = std::conditional_t<std::is_void_v<R>, std::common_type_t<A, B>, R>;
  return shim_internal::UniformImpl<T>(g, static_cast<T>(lo), static_cast<T>(hi), false);
}
template <typename R = void, typename G, typename A, typename B>
auto Uniform(IntervalClosedClosedTag, G&& g, A lo, B hi) {
  using T = std::conditional_t<std::is_void_v<R>, std::common_type_t<A, B>, R>;
  return shim_internal::UniformImpl<T>(g, static_cast<T>(lo), static_cast<T>(hi), true);
}
template <typename R = void, typename G, typename A, typename B>
auto Uniform(IntervalClosedOpenTag, G&& g, A lo, B hi) {
  using T = std::conditional_t<std::is_void_v<R>, std::common_type_t<A, B>, R>;
  return shim_internal::UniformImpl<T>(g, static_cast<T>(lo), static_cast<T>(hi), false);
}
template <typename R, typename G>
R Uniform(G&& g) { return uniform_int_distribution<R>((std::numeric_limits<R>::min)(), (std::numeric_limits<R>::max)())(g); }
template <typename G>
bool Bernoulli(G&& g, double p) { return uniform_real_distribution<double>(0.0, 1.0)(g) < p; }

class BitGen {
 public:
  using result_type = uint64_t;
  BitGen() : g_(std::random_device{}()) {}
  static constexpr result_type min() { return 0; }
  static constexpr result_type max() { return ~0ull; }
  result_type operator()() { return g_(); }
 private:
  std::mt19937_64 g_;
};
using InsecureBitGen = BitGen;

class BitGenRef {
 public:
  using result_type = uint64_t;
  template <typename G, typename = std::enable_if_t<!std::is_same_v<std::decay_t<G>, BitGenRef>>>
  BitGenRef(G& g) : p_(&g), f_([](void* p) -> uint64_t { return shim_internal::FastBits<uint64_t>(*static_cast<G*>(p)); }) {}
  BitGenRef(const BitGenRef&) = default;
  static constexpr result_type min() { return 0; }
  static constexpr result_type max() { return ~0ull; }
  result_type operator()() { return f_(p_); }
 private:
  void* p_;
  uint64_t (*f_)(void*);
};

}  // namespace absl
#endif  // B2S_ABSL_SHIM_ALL_H_
