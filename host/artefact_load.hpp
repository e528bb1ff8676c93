// artefact_load.hpp — reads an RMI back from the artefacts codegen.hpp (and the reference's codegen.rs) writes:
//   <out_dir>/<ns>.cpp, <ns>.h, <ns>_data.h and <data_dir>/<ns>_L{i}_PARAMETERS
// and rebuilds the two-layer model, its error bounds when the artefact carries them, and for a `--bounded` artefact
// the cache-fix knots, line size and total key count.  Host code only; compiles with g++ like codegen.hpp.
//
// Accepted are exactly the forms the generator emits (codegen.rs LayerParams: Constant / Array / MixedArray):
//   - constants in <ns>_data.h: floats in Rust's Display form (NaN, inf, long positional digits; strtod reads them
//     back exactly) with c_val()'s ".0", integers as 123UL, inline arrays as { 1UL, 2UL } (a radix8 table);
//   - blobs, whose byte count is the one load() reads (`infile.read((char*)L1_PARAMETERS, <bytes>)`), never more;
//   - the models, named by the functions lookup() calls.  linear, robust_linear and linear_spline emit the same
//     function `linear`, so all three load as linear (RMI_MODEL_LINEAR): their predictions are identical.
// The reference writes its declaration blocks in HashSet order; nothing here depends on the order of those lines.
// Errors are LoadError: RMI_ERR_INVALID for a malformed artefact (the message names the file), RMI_ERR_UNSUPPORTED
// for a `--bounded` artefact without errors, whose generated code calls _rmi_lookup_pre_cachefix with an argument
// it does not declare.
#pragma once
#include <cerrno>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../include/rmi_b200.h"
#include "cache_fix.hpp"
#include "codegen.hpp"

namespace rmihost {

struct LoadError : std::runtime_error {
  int code;
  LoadError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

// A loaded RMI: `r` points into the vectors below (valid while this object lives and is not copied).
struct LoadedArtefact {
  rmi_result r{};
  std::vector<double> params;
  std::vector<uint64_t> errors;
  std::vector<uint32_t> t32;
  std::vector<uint64_t> a1, a2;
  int key_type = RMI_KEY_U64;
  bool has_errors = false;
  uint64_t line_size = 0, total_keys = 0, build_time_ns = 0;
  std::vector<SplinePoint> knots;
  LoadedArtefact() = default;
  LoadedArtefact(const LoadedArtefact&) = delete;
  LoadedArtefact& operator=(const LoadedArtefact&) = delete;
};

namespace artefact_detail {

[[noreturn]] inline void bad(const std::string& file, const std::string& what) {
  throw LoadError(RMI_ERR_INVALID, file + ": " + what);
}

inline std::vector<std::string> read_lines(const std::string& path) {
  std::ifstream in(path);
  if (!in) bad(path, "cannot be read");
  std::vector<std::string> lines;
  for (std::string s; std::getline(in, s);) lines.push_back(s);
  return lines;
}

inline bool starts_with(const std::string& s, const std::string& p) { return s.compare(0, p.size(), p) == 0; }
inline std::string trim(const std::string& s) {
  size_t a = s.find_first_not_of(" \t\r"), b = s.find_last_not_of(" \t\r");
  return a == std::string::npos ? std::string() : s.substr(a, b - a + 1);
}
// The text between `pre` and the next `post` in s (after `pre`); false if either is missing.
inline bool between(const std::string& s, const std::string& pre, const std::string& post, std::string* out) {
  size_t a = s.find(pre);
  if (a == std::string::npos) return false;
  a += pre.size();
  size_t b = s.find(post, a);
  if (b == std::string::npos) return false;
  *out = s.substr(a, b - a);
  return true;
}

inline uint64_t parse_u64(const std::string& file, const std::string& t, const char* suffix = "") {
  const size_t sl = std::strlen(suffix);
  if (t.size() <= sl || t.compare(t.size() - sl, sl, suffix) != 0) bad(file, "bad integer constant '" + t + "'");
  const std::string digits = t.substr(0, t.size() - sl);
  if (digits.empty() || digits.find_first_not_of("0123456789") != std::string::npos || digits.size() > 20)
    bad(file, "bad integer constant '" + t + "'");
  errno = 0;
  char* end = nullptr;
  const unsigned long long v = std::strtoull(digits.c_str(), &end, 10);
  if (errno == ERANGE || *end) bad(file, "bad integer constant '" + t + "'");
  return v;
}

// c_val() of a float (codegen.hpp): Rust Display digits, ".0" appended where no '.' is present.
inline double parse_f64(const std::string& file, const std::string& t) {
  if (t == "NaN.0") return std::nan("");
  if (t == "inf.0") return INFINITY;
  if (t == "-inf.0") return -INFINITY;
  if (t.empty() || t.find('.') == std::string::npos || t.find_first_not_of("-0123456789.") != std::string::npos)
    bad(file, "bad float constant '" + t + "'");
  char* end = nullptr;
  const double v = std::strtod(t.c_str(), &end);
  if (*end || std::isnan(v)) bad(file, "bad float constant '" + t + "'");
  return v;
}

// `{ 1UL, 2UL }`
inline std::vector<uint64_t> parse_u64_list(const std::string& file, const std::string& t) {
  if (t.size() < 4 || t.compare(0, 2, "{ ") != 0 || t.compare(t.size() - 2, 2, " }") != 0) bad(file, "bad array constant");
  std::vector<uint64_t> v;
  std::stringstream ss(t.substr(2, t.size() - 4));
  for (std::string item; std::getline(ss, item, ',');) v.push_back(parse_u64(file, trim(item), "UL"));
  return v;
}

struct DataHeader {
  struct Constant { std::string type, value; bool array; };
  std::map<std::string, Constant> constants;   // L<i>_PARAMETER<p>
  std::map<std::string, std::string> arrays;   // L<i>_PARAMETERS -> element type (char for a mixed layer)
};

inline void check_namespace(const std::string& file, const std::string& line, const std::string& ns) {
  if (line != "namespace " + ns + " {") bad(file, "namespace does not match '" + ns + "'");
}

inline DataHeader parse_data_header(const std::string& file, const std::string& ns) {
  DataHeader d;
  bool seen_ns = false;
  for (const std::string& raw : read_lines(file)) {
    const std::string line = trim(raw);
    if (line.empty() || line == "} // namespace") continue;
    if (starts_with(line, "namespace ")) { check_namespace(file, line, ns); seen_ns = true; continue; }
    if (starts_with(line, "const ")) {   // const <type> <name>[[]] = <value>;
      const size_t sp = line.find(' ', 6), eq = line.find(" = ");
      if (sp == std::string::npos || eq == std::string::npos || eq < sp || line.back() != ';') bad(file, "bad line '" + line + "'");
      std::string name = line.substr(sp + 1, eq - sp - 1);
      DataHeader::Constant c{line.substr(6, sp - 6), line.substr(eq + 3, line.size() - eq - 4), false};
      if (name.size() > 2 && name.compare(name.size() - 2, 2, "[]") == 0) { c.array = true; name.resize(name.size() - 2); }
      d.constants[name] = c;
      continue;
    }
    // <type>* L<i>_PARAMETERS;  or  <type> L<i>_PARAMETERS[<items>];
    const size_t sp = line.find(' ');
    if (sp == std::string::npos || line.back() != ';') bad(file, "bad line '" + line + "'");
    std::string type = line.substr(0, sp), name = line.substr(sp + 1, line.size() - sp - 2);
    if (!type.empty() && type.back() == '*') type.pop_back();
    const size_t br = name.find('[');
    if (br != std::string::npos) name.resize(br);
    if (!starts_with(name, "L") || name.find("_PARAMETERS") == std::string::npos) bad(file, "bad line '" + line + "'");
    d.arrays[name] = type;
  }
  if (!seen_ns) bad(file, "no namespace");
  return d;
}

struct ModelFn { const char* name; int kind; int high; size_t params; bool float_out; };
inline const ModelFn* model_fn(const std::string& name) {
  static const ModelFn fns[] = {
      {"linear", RMI_MODEL_LINEAR, 1, 2, true},     {"cubic", RMI_MODEL_CUBIC, 1, 4, true},
      {"loglinear", RMI_MODEL_LOGLINEAR, 1, 2, true}, {"ncdf", RMI_MODEL_NORMAL, 1, 3, true},
      {"lncdf", RMI_MODEL_LOGNORMAL, 1, 3, true},   {"radix", RMI_MODEL_RADIX, 1, 2, false},
      {"radix_table", RMI_MODEL_RADIX_TABLE, 1, 1, false}, {"bradix_clamp_high", RMI_MODEL_BRADIX, 1, 3, false},
      {"bradix_clamp_low", RMI_MODEL_BRADIX, 0, 3, false}, {"ed_histogram", RMI_MODEL_HISTOGRAM, 1, 3, false}};
  for (const auto& f : fns) if (name == f.name) return &f;
  return nullptr;
}

// `  fpred = name(args);` -> name
inline std::string call_name(const std::string& file, const std::string& line) {
  std::string name;
  if (!between(line, "pred = ", "(", &name)) bad(file, "bad model call '" + trim(line) + "'");
  return name;
}

// FCLAMP(fpred, <b>.0 - 1.0)  or  (ipred > <b> - 1 ? <b> - 1 : ipred) -> b; 0 where no bound is printed
inline uint64_t clamp_bound(const std::string& file, const std::string& expr) {
  std::string b;
  if (between(expr, "FCLAMP(fpred, ", ".0 - 1.0)", &b)) return parse_u64(file, b);
  if (between(expr, "(ipred > ", " - 1 ?", &b)) return parse_u64(file, b);
  return 0;
}

inline std::vector<char> read_blob(const std::string& path, uint64_t bytes) {
  std::ifstream in(path, std::ios::binary);
  if (!in) bad(path, "missing");
  in.seekg(0, std::ios::end);
  const std::streamoff size = in.tellg();
  if (size < 0 || (uint64_t)size < bytes)
    bad(path, "truncated: " + std::to_string(size < 0 ? 0 : (long long)size) + " bytes, load() reads " + std::to_string(bytes));
  in.seekg(0);
  std::vector<char> buf(bytes);
  if (bytes && !in.read(buf.data(), (std::streamsize)bytes)) bad(path, "read failed");
  return buf;
}

}  // namespace artefact_detail

// Loads <out_dir>/<ns>.{cpp,h,_data.h} and the blobs under data_dir into *out.
inline void load_rmi(const std::string& ns, const std::string& out_dir, const std::string& data_dir, LoadedArtefact* out) {
  using namespace artefact_detail;
  LoadedArtefact& A = *out;
  const std::string f_cpp = out_dir + "/" + ns + ".cpp", f_h = out_dir + "/" + ns + ".h", f_data = out_dir + "/" + ns + "_data.h";

  // ---- <ns>.h: RMI_SIZE, BUILD_TIME_NS, NAME ----------------------------------------------------------------------
  uint64_t rmi_size_h = 0;
  bool have_size = false, have_time = false, have_name = false, seen_ns = false;
  for (const std::string& line : read_lines(f_h)) {
    std::string v;
    if (starts_with(line, "namespace ")) { check_namespace(f_h, line, ns); seen_ns = true; }
    else if (between(line, "const size_t RMI_SIZE = ", ";", &v)) { rmi_size_h = parse_u64(f_h, v); have_size = true; }
    else if (between(line, "const uint64_t BUILD_TIME_NS = ", ";", &v)) { A.build_time_ns = parse_u64(f_h, v); have_time = true; }
    else if (between(line, "const char NAME[] = \"", "\";", &v)) {
      if (v != ns) bad(f_h, "NAME is '" + v + "', not '" + ns + "'");
      have_name = true;
    }
  }
  if (!seen_ns || !have_size || !have_time || !have_name) bad(f_h, "RMI_SIZE, BUILD_TIME_NS, NAME or the namespace missing");

  const DataHeader dh = parse_data_header(f_data, ns);

  // ---- <ns>.cpp: blob sizes from load(), the lookup body, function texts ---------------------------------------------
  const std::vector<std::string> cpp = read_lines(f_cpp);
  std::map<std::string, uint64_t> blob_bytes;   // L<i>_PARAMETERS -> bytes load() reads
  std::map<std::string, std::string> blob_file; // L<i>_PARAMETERS -> file name under data_dir
  size_t rmi_fn = cpp.size(), spline_fn = cpp.size();
  std::string rmi_sig;
  bool seen_cpp_ns = false;
  unsigned radix_prefix = 0, radix_nb = 0;
  bool have_radix_text = false;
  for (size_t i = 0; i < cpp.size(); ++i) {
    const std::string& line = cpp[i];
    std::string v;
    if (starts_with(line, "namespace ")) { check_namespace(f_cpp, line, ns); seen_cpp_ns = true; }
    else if (between(line, "std::filesystem::path(dataPath) / \"", "\"", &v)) {
      const std::string pre = ns + "_";
      if (!starts_with(v, pre)) bad(f_cpp, "blob '" + v + "' is not in namespace '" + ns + "'");
      blob_file[v.substr(pre.size())] = v;
    } else if (between(line, "infile.read((char*)", ");", &v)) {
      const size_t c = v.find(", ");
      if (c == std::string::npos) bad(f_cpp, "bad load() line '" + trim(line) + "'");
      blob_bytes[v.substr(0, c)] = parse_u64(f_cpp, v.substr(c + 2));
    } else if (starts_with(line, "uint64_t _rmi_lookup_pre_cachefix(")) { rmi_fn = i; rmi_sig = line; }
    else if (starts_with(line, "uint64_t lookup(")) {
      if (rmi_fn == cpp.size() || rmi_sig.find("_rmi_lookup_pre_cachefix") == std::string::npos) { rmi_fn = i; rmi_sig = line; }
      else spline_fn = i;
    } else if (starts_with(line, "inline uint64_t radix_table(") && i + 1 < cpp.size()) {
      std::string p, nb;
      if (!between(cpp[i + 1], "return table[((inp << ", ") >> ", &p) || !between(cpp[i + 1], ") >> " + p + ") >> ", "];", &nb))
        bad(f_cpp, "bad radix_table function");
      radix_prefix = (unsigned)parse_u64(f_cpp, p);
      radix_nb = (unsigned)parse_u64(f_cpp, nb);
      have_radix_text = true;
    }
  }
  if (!seen_cpp_ns) bad(f_cpp, "no namespace");
  if (rmi_fn == cpp.size()) bad(f_cpp, "no lookup function");
  const bool bounded = rmi_sig.find("_rmi_lookup_pre_cachefix") != std::string::npos;
  // signature: uint64_t <fn>(<key type> key[, size_t* err]) {
  std::string ktype;
  if (!between(rmi_sig, "(", " key", &ktype)) bad(f_cpp, "bad lookup signature");
  if (ktype == "uint64_t") A.key_type = RMI_KEY_U64;
  else if (ktype == "double") A.key_type = RMI_KEY_F64;
  else bad(f_cpp, "unknown key type '" + ktype + "'");
  A.has_errors = rmi_sig.find("size_t* err") != std::string::npos;
  if (bounded && !A.has_errors)
    throw LoadError(RMI_ERR_UNSUPPORTED, f_cpp + ": a --bounded RMI without errors (its generated code does not compile: "
                                                 "_rmi_lookup_pre_cachefix is called with an error argument it does not declare)");
  if (bounded && spline_fn == cpp.size()) bad(f_cpp, "no cache-fix lookup");

  // the RMI's body: the two model calls, the model index, the error line and the final clamp
  std::vector<std::string> calls;
  std::string model_index, err_line, ret;
  for (size_t i = rmi_fn + 1; i < cpp.size() && cpp[i] != "}"; ++i) {
    const std::string line = trim(cpp[i]);
    if (starts_with(line, "fpred = ") || starts_with(line, "ipred = ")) calls.push_back(line);
    else if (starts_with(line, "modelIndex = ")) model_index = line;
    else if (starts_with(line, "*err = ")) err_line = line;
    else if (starts_with(line, "return ")) ret = line;
  }
  if (calls.size() != 2 || ret.empty()) bad(f_cpp, "lookup body does not hold two model calls and a return");
  const ModelFn* top = model_fn(call_name(f_cpp, calls[0]));
  const ModelFn* leaf = model_fn(call_name(f_cpp, calls[1]));
  if (!top) bad(f_cpp, "unknown top model function '" + call_name(f_cpp, calls[0]) + "'");
  if (!leaf || !leaf->float_out) bad(f_cpp, "unknown leaf model function '" + call_name(f_cpp, calls[1]) + "'");
  const uint64_t rows = clamp_bound(f_cpp, ret);
  if (rows == 0) bad(f_cpp, "no row count in '" + ret + "'");

  auto constant = [&](int layer, size_t p) -> const DataHeader::Constant& {
    const std::string name = "L" + std::to_string(layer) + "_PARAMETER" + std::to_string(p);
    auto it = dh.constants.find(name);
    if (it == dh.constants.end()) bad(f_data, name + " missing");
    return it->second;
  };
  auto float_constant = [&](int layer, size_t p) {
    const auto& c = constant(layer, p);
    if (c.type != "double" || c.array) bad(f_data, "L" + std::to_string(layer) + " parameter " + std::to_string(p) + " is not a double");
    return parse_f64(f_data, c.value);
  };
  auto int_constant = [&](int layer, size_t p) {
    const auto& c = constant(layer, p);
    if (c.type != "uint64_t" || c.array) bad(f_data, "L" + std::to_string(layer) + " parameter " + std::to_string(p) + " is not a uint64_t");
    return parse_u64(f_data, c.value, "UL");
  };
  // a layer's blob: declared in _data.h, read by load(), present in data_dir with at least that many bytes
  auto blob = [&](const std::string& name, const char* type) -> std::vector<char> {
    auto d = dh.arrays.find(name);
    if (d == dh.arrays.end()) bad(f_data, name + " not declared");
    if (d->second != type) bad(f_data, name + " has element type " + d->second + ", expected " + type);
    auto b = blob_bytes.find(name);
    auto f = blob_file.find(name);
    if (b == blob_bytes.end() || f == blob_file.end()) bad(f_cpp, "load() does not read " + name);
    return read_blob(data_dir + "/" + f->second, b->second);
  };
  auto u64_at = [](const std::vector<char>& b, size_t k) { uint64_t v; std::memcpy(&v, b.data() + 8 * k, 8); return v; };

  // ---- layer 0 ------------------------------------------------------------------------------------------------------
  rmi_result& r = A.r;
  std::memset(&r, 0, sizeof(r));
  r.l0_model_id = (uint32_t)top->kind;
  r.l0_bradix_high = (uint32_t)top->high;
  if (top->float_out) {
    r.l0_num_fparams = (uint32_t)top->params;
    for (size_t p = 0; p < top->params; ++p) r.l0_fparams[p] = float_constant(0, p);
  } else if (top->kind == RMI_MODEL_RADIX || top->kind == RMI_MODEL_BRADIX) {
    r.l0_num_iparams = (uint32_t)top->params;
    for (size_t p = 0; p < top->params; ++p) r.l0_iparams[p] = int_constant(0, p);
  } else if (top->kind == RMI_MODEL_RADIX_TABLE) {
    if (dh.arrays.count("L0_PARAMETERS")) {
      std::vector<char> b = blob("L0_PARAMETERS", "uint32_t");
      if (b.size() % 4) bad(f_cpp, "L0_PARAMETERS: byte count not a multiple of 4");
      A.t32.resize(b.size() / 4);
      std::memcpy(A.t32.data(), b.data(), b.size());
    } else {
      const auto& c = constant(0, 0);
      if (c.type != "uint32_t" || !c.array) bad(f_data, "L0_PARAMETER0 is not a uint32_t array");
      for (uint64_t v : parse_u64_list(f_data, c.value)) {
        if (v > 0xffffffffull) bad(f_data, "radix table entry out of range");
        A.t32.push_back((uint32_t)v);
      }
    }
    unsigned bits = 0;
    while (bits < 32 && ((size_t)1 << bits) < A.t32.size()) ++bits;
    if (A.t32.empty() || ((size_t)1 << bits) != A.t32.size()) bad(f_data, "radix table length is not a power of two");
    if (!have_radix_text) bad(f_cpp, "radix_table function missing");
    const unsigned nb = radix_prefix + bits > 64 ? 0 : 64 - (radix_prefix + bits);
    if (nb != radix_nb) bad(f_cpp, "radix_table shift does not match the table length");
    r.l0_table_bits = bits;
    r.l0_num_iparams = 1;
    r.l0_iparams[0] = radix_prefix;
  } else {   // histogram: mixed blob {len, radix index, pivots}
    std::vector<char> b = blob("L0_PARAMETERS", "char");
    if (b.size() < 8 || b.size() % 8) bad(f_cpp, "L0_PARAMETERS: bad histogram byte count");
    const uint64_t words = b.size() / 8, len = u64_at(b, 0);
    if (len == 0 || len > words - 1) bad(f_cpp, "L0_PARAMETERS: histogram length does not fit the blob");
    const uint64_t ri = words - 1 - len;
    A.a1.resize(ri);
    A.a2.resize(len);
    std::memcpy(A.a1.data(), b.data() + 8, 8 * ri);
    std::memcpy(A.a2.data(), b.data() + 8 * (1 + ri), 8 * len);
    r.l0_num_iparams = 1;
    r.l0_iparams[0] = len;
  }

  // ---- layer 1 ------------------------------------------------------------------------------------------------------
  const size_t ppm = leaf->params;
  uint64_t N = 0;
  if (dh.arrays.count("L1_PARAMETERS")) {
    std::vector<char> b = blob("L1_PARAMETERS", A.has_errors ? "char" : "double");
    const size_t rec = 8 * (ppm + (A.has_errors ? 1 : 0));
    if (b.empty() || b.size() % rec) bad(f_cpp, "L1_PARAMETERS: " + std::to_string(b.size()) + " bytes is not a whole number of " +
                                              std::to_string(rec) + "-byte leaf records");
    N = b.size() / rec;
    A.params.resize(N * ppm);
    if (A.has_errors) A.errors.resize(N);
    for (uint64_t j = 0; j < N; ++j) {
      std::memcpy(&A.params[j * ppm], b.data() + j * rec, 8 * ppm);
      if (A.has_errors) A.errors[j] = u64_at(b, j * (ppm + 1) + ppm);
    }
  } else {
    N = 1;
    for (size_t p = 0; p < ppm; ++p) A.params.push_back(float_constant(1, p));
    if (A.has_errors) {
      std::string v;
      if (!between(err_line, "*err = ", ";", &v)) bad(f_cpp, "no error bound in the lookup");
      A.errors.push_back(parse_u64(f_cpp, v));
    }
  }
  if (N > 1) {
    if (model_index.empty()) bad(f_cpp, "no model index in the lookup");
    const uint64_t printed = clamp_bound(f_cpp, model_index);
    if (printed && printed != N) bad(f_cpp, "the model index clamps at " + std::to_string(printed) + ", L1_PARAMETERS holds " +
                                            std::to_string(N) + " leaves");
  }
  r.branching_factor = N;
  r.num_rmi_rows = rows;
  r.l1_model_id = (uint32_t)leaf->kind;
  r.l1_params_per_model = (uint32_t)ppm;

  // ---- the cache-fix spline of a --bounded artefact --------------------------------------------------------------
  CacheFixInfo cf;
  if (bounded) {
    std::string pts, total, ls, arr;
    for (size_t i = spline_fn + 1; i < cpp.size() && cpp[i] != "}"; ++i) {
      std::string v;
      if (between(cpp[i], "const uint64_t num_spline_pts = ", ";", &v)) pts = v;
      else if (between(cpp[i], "const uint64_t total_keys = ", ";", &v)) total = v;
      else if (between(cpp[i], "*err = ", ";", &v)) ls = v;
      else if (between(cpp[i], "(struct SplinePoint*) ", ";", &v)) arr = v;
    }
    if (pts.empty() || total.empty() || ls.empty() || arr.empty()) bad(f_cpp, "incomplete cache-fix lookup");
    const uint64_t K = parse_u64(f_cpp, pts);
    A.total_keys = parse_u64(f_cpp, total);
    A.line_size = parse_u64(f_cpp, ls);
    std::vector<char> b = blob(arr, "uint64_t");
    if (b.size() != 16 * K) bad(f_cpp, arr + ": " + std::to_string(b.size()) + " bytes for " + std::to_string(K) + " spline points");
    if (K != rows) bad(f_cpp, "the RMI covers " + std::to_string(rows) + " rows, the spline has " + std::to_string(K) + " points");
    A.knots.resize(K);
    for (uint64_t k = 0; k < K; ++k) A.knots[k] = SplinePoint(u64_at(b, 2 * k), u64_at(b, 2 * k + 1));
    cf.line_size = A.line_size;
    cf.spline = &A.knots;
    cf.num_data_rows = A.total_keys;
  }

  // ---- pointers, statistics (not in the artefact), cross-check of the header's size -----------------------------
  r.num_data_rows = bounded ? A.total_keys : rows;
  r.l0_table32_len = A.t32.size();
  r.l0_table32 = A.t32.empty() ? nullptr : A.t32.data();
  r.l0_array1_len = A.a1.size();
  r.l0_array1 = A.a1.empty() ? nullptr : A.a1.data();
  r.l0_array2_len = A.a2.size();
  r.l0_array2 = A.a2.empty() ? nullptr : A.a2.data();
  r.l1_params = A.params.data();
  r.l1_errors = A.has_errors ? A.errors.data() : nullptr;
  r.model_avg_error = r.model_avg_l2_error = r.model_avg_log2_error = r.model_max_log2_error = std::nan("");
  r.build_time_ns = A.build_time_ns;
  const uint64_t size = rmi_size(r, A.has_errors, bounded ? &cf : nullptr);
  if (size != rmi_size_h)
    bad(f_h, "RMI_SIZE is " + std::to_string(rmi_size_h) + ", the loaded model has " + std::to_string(size) + " bytes");
}

}  // namespace rmihost
