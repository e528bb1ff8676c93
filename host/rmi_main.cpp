// rmi — command-line front end with the reference's argument surface (src/main.rs:36-102):
//   rmi <input> [namespace] [models] [branching factor]
//       [--no-code] [--param-grid <file>] [--data-path|-d <dir>] [--no-errors] [--threads|-t <n>]
//       [--max-size <bytes>] [--disable-parallel-training] [--zero-build-time] [--optimize <file>]
//       [--bounded <line_size>]
// plus  --exact-top-fit (RMI_FLAG_TOP_FIT_EXACT), --device <n> and, for the configuration sweeps
// (--optimize, --max-size), --devices <a,b,...>: the key set is replicated to every listed GPU
// (device-to-device copies) and the independent configurations are spread over them.
// The build itself is librmi_b200.so (CUDA); this binary only loads the data set into HBM,
// calls rmi_train and writes the artefacts (codegen.hpp).  `--bounded` fits the reference's
// cache-fix spline on the GPU from the loaded keys (rmi_cache_fix_device) and then builds the RMI
// over the spline's knots on the GPU like any other data set.  There is no CPU training path: without a usable
// GPU every build fails with the CUDA error text.
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "../include/rmi_b200.h"
#include "codegen.hpp"
#include "optimizer.hpp"
#include "param_grid.hpp"

using namespace rmihost;

namespace {

[[noreturn]] void die(const std::string& msg) {
  std::fprintf(stderr, "rmi: %s\n", msg.c_str());
  std::exit(101);   // the exit status of a Rust panic
}

struct Args {
  std::vector<std::string> pos;
  std::map<std::string, std::string> opt;
  bool has(const std::string& k) const { return opt.count(k) != 0; }
};

Args parse_args(int argc, char** argv) {
  const std::map<std::string, bool> takes_value = {
      {"--no-code", false}, {"--dump-ll-model-data", true}, {"--dump-ll-errors", false}, {"--stats-file", true},
      {"--param-grid", true}, {"--data-path", true}, {"--no-errors", false}, {"--threads", true}, {"--bounded", true},
      {"--max-size", true}, {"--disable-parallel-training", false}, {"--zero-build-time", false}, {"--optimize", true},
      {"--exact-top-fit", false}, {"--device", true}, {"--devices", true}, {"--verbose", false}};
  Args a;
  for (int i = 1; i < argc; ++i) {
    std::string s = argv[i];
    if (s == "-d") s = "--data-path";
    if (s == "-t") s = "--threads";
    if (s == "-s") s = "--stats-file";
    if (s.rfind("--", 0) == 0) {
      std::string key = s, val;
      size_t eq = s.find('=');
      if (eq != std::string::npos) { key = s.substr(0, eq); val = s.substr(eq + 1); }
      auto it = takes_value.find(key);
      if (it == takes_value.end()) die("error: Found argument '" + key + "' which wasn't expected");
      if (it->second && eq == std::string::npos) { if (i + 1 >= argc) die("error: " + key + " requires a value"); val = argv[++i]; }
      a.opt[key] = val;
    } else a.pos.push_back(s);
  }
  return a;
}

void print_stats(const rmi_result& r, uint64_t num_rows) {   // main.rs:297-321 (info! lines)
  std::fprintf(stderr, "Model build time: %llu ms\n", (unsigned long long)(r.build_time_ns / 1000000));
  std::fprintf(stderr, "Average model error: %g (%g%%)\n", r.model_avg_error, r.model_avg_error / (double)num_rows * 100.0);
  std::fprintf(stderr, "Average model L2 error: %g\n", r.model_avg_l2_error);
  std::fprintf(stderr, "Average model log2 error: %g\n", r.model_avg_log2_error);
  std::fprintf(stderr, "Max model log2 error: %g\n", r.model_max_log2_error);
  std::fprintf(stderr, "Max model error on model %llu: %llu (%g%%)\n", (unsigned long long)r.model_max_error_idx,
               (unsigned long long)r.model_max_error, (double)r.model_max_error / (double)num_rows * 100.0);
}

}  // namespace

int main(int argc, char** argv) {
  Args a = parse_args(argc, argv);
  if (a.pos.empty()) die("error: The following required arguments were not provided:\n    <input>");
  const std::string fp = a.pos[0];
  const std::string data_dir = a.has("--data-path") ? a.opt["--data-path"] : "rmi_data";
  const bool have_ns = a.pos.size() > 1;
  if (have_ns && a.has("--param-grid")) die("Can only specify one of namespace or param-grid");
  const int device = a.has("--device") ? std::atoi(a.opt["--device"].c_str())
                                       : (a.has("--devices") ? std::atoi(a.opt["--devices"].c_str()) : 0);
  const uint32_t flags = a.has("--exact-top-fit") ? RMI_FLAG_TOP_FIT_EXACT : 0;
  const bool verbose = a.has("--verbose") || std::getenv("RUST_LOG") != nullptr;

  // main.rs:121-132: the key type comes from the file NAME
  int file_kt;
  int code_kt = RMI_KEY_U64;   // KeyType handed to codegen: uint32 files keep U64
  if (fp.find("uint64") != std::string::npos) file_kt = RMI_KEY_U64;
  else if (fp.find("uint32") != std::string::npos) file_kt = RMI_KEY_U32;
  else if (fp.find("f64") != std::string::npos) { file_kt = RMI_KEY_F64; code_kt = RMI_KEY_F64; }
  else die("Data file must contain uint64, uint32, or f64.");

  rmi_dataset* ds = nullptr;
  if (rmi_dataset_load_file(fp.c_str(), file_kt, device, &ds) != RMI_OK) die(rmi_last_error());
  const uint64_t num_rows = rmi_dataset_len(ds);

  // replicas of the key set for the sweeps: the first listed device holds the loaded copy
  std::vector<const rmi_dataset*> replicas{ds};
  std::vector<rmi_dataset*> owned_replicas;
  if (a.has("--devices") && (a.has("--optimize") || a.has("--max-size"))) {
    // one worker thread per listed device; a device listed more than once gets more workers on the SAME
    // resident copy (the data set is immutable and rmi_train is re-entrant), other devices get a replica
    std::stringstream dl(a.opt["--devices"]);
    std::string tok;
    std::map<int, const rmi_dataset*> on_device{{device, ds}};
    bool loaded_counted = false;
    while (std::getline(dl, tok, ',')) {
      if (tok.empty()) continue;
      int d = std::atoi(tok.c_str());
      // the loaded copy already has its worker (replicas[0]): the FIRST mention of its device, wherever it
      // stands in the list, is that worker; further mentions add workers on the same resident copy
      if (d == device && !loaded_counted) { loaded_counted = true; continue; }
      auto it = on_device.find(d);
      if (it == on_device.end()) {
        rmi_dataset* rep = nullptr;
        if (rmi_dataset_replicate(ds, d, &rep) != RMI_OK) die(rmi_last_error());
        owned_replicas.push_back(rep);
        it = on_device.emplace(d, rep).first;
      }
      replicas.push_back(it->second);
    }
  }
  auto free_replicas = [&]() { for (auto* r : owned_replicas) rmi_dataset_destroy(r); owned_replicas.clear(); };

  if (a.has("--optimize")) {   // main.rs:134-161
    std::vector<RMIStatistics> results;
    try { results = find_pareto_efficient_configs(replicas, 10, flags, verbose); } catch (std::exception& e) { die(e.what()); }
    free_replicas();
    display_table(results);
    std::string prefix;
    if (have_ns) prefix = a.pos[1];
    else { size_t sl = fp.find_last_of('/'); prefix = sl == std::string::npos ? fp : fp.substr(sl + 1); }
    std::ofstream out(a.opt["--optimize"]);
    if (!out) die("Could not write optimization results file");
    out << "{\"configs\":[";
    for (size_t i = 0; i < results.size(); ++i) {
      auto& v = results[i];
      if (i) out << ",";
      out << "{\"layers\":" << json_str(v.models) << ",\"branching factor\":" << v.branching_factor << ",\"namespace\":"
          << json_str(prefix + "_" + std::to_string(i)) << ",\"size\":" << v.size << ",\"average log2 error\":"
          << json_num(v.average_log2_error) << ",\"binary\":true}";
    }
    out << "]}";
    rmi_dataset_destroy(ds);
    return 0;
  }

  {   // main.rs:164-169: create_dir_all
    std::error_code ec;
    if (!std::filesystem::exists(data_dir, ec)) {
      std::filesystem::create_directories(data_dir, ec);
      if (ec) die("The RMI data directory did not exist, and it could not be created.");
    }
  }

  auto train_one = [&](const std::string& models, uint64_t bf, rmi_result** out) {
    if (rmi_train(ds, models.c_str(), bf, flags, out) != RMI_OK) die(rmi_last_error());
  };

  if (a.has("--param-grid")) {   // main.rs:171-261
    std::ifstream in(a.opt["--param-grid"]);
    if (!in) die("could not read the parameter grid file");
    std::stringstream ss; ss << in.rdbuf();
    std::vector<GridEntry> grid;
    try { grid = parse_param_grid(ss.str()); } catch (std::exception& e) { die(e.what()); }
    std::ofstream out(a.opt["--param-grid"] + "_results");
    if (!out) die("Could not write results file");
    std::vector<GridResult> results;
    for (auto& g : grid) {   // one GPU executes builds back to back: the grid is walked in order
      rmi_result* r = nullptr;
      train_one(g.layers, g.branching_factor, &r);
      GridResult gr;
      gr.entry = g;
      gr.avg_error = r->model_avg_error; gr.avg_l2 = r->model_avg_l2_error; gr.avg_log2 = r->model_avg_log2_error;
      gr.max_log2 = r->model_max_log2_error; gr.max_error = r->model_max_error; gr.size_bs = rmi_size(*r, true);
      results.push_back(gr);
      if (g.has_namespace) {
        try { output_rmi(g.ns, *r, data_dir, code_kt, true, a.has("--zero-build-time") ? 0 : r->build_time_ns); }
        catch (std::exception& e) { die(e.what()); }
      }
      rmi_result_free(r);
    }
    out << grid_results_json(results, num_rows);
  } else if (have_ns) {   // main.rs:263-333
    const std::string ns = a.pos[1];
    rmi_result* r = nullptr;
    CacheFixInfo cf;
    std::vector<SplinePoint> spline;
    bool bounded = false, sized = false;
    uint64_t bounded_build_ns = 0;
    if (a.has("--max-size")) {   // train_for_size, train/mod.rs:128-154
      uint64_t max_size = std::strtoull(a.opt["--max-size"].c_str(), nullptr, 10);
      auto t0 = std::chrono::steady_clock::now();   // train_for_size times the sweep AND the final build (train/mod.rs:131-152)
      std::vector<RMIStatistics> pareto;
      try { pareto = find_pareto_efficient_configs(replicas, 1000, flags, verbose); } catch (std::exception& e) { die(e.what()); }
      free_replicas();
      const RMIStatistics* pick = nullptr;
      for (auto& c : pareto) if (c.size < max_size) { pick = &c; break; }
      if (!pick) die("Could not find any configurations smaller than " + std::to_string(max_size));
      std::fprintf(stderr, "Found RMI config %s %llu with size %llu and average log2 %g\n", pick->models.c_str(),
                   (unsigned long long)pick->branching_factor, (unsigned long long)pick->size, pick->average_log2_error);
      train_one(pick->models, pick->branching_factor, &r);
      bounded_build_ns = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      sized = true;
    } else if (a.has("--bounded")) {
      // train_bounded (train/mod.rs:156-184): the cache-fix spline fitted on the device from the keys already
      // loaded, then the ordinary GPU build with the spline's knots as the data set (their offsets are 0, 1, 2, ...)
      if (a.pos.size() < 4) die("called `Option::unwrap()` on a `None` value (models and branching factor are required)");
      char* endp = nullptr;
      const std::string ls = a.opt["--bounded"];
      cf.line_size = std::strtoull(ls.c_str(), &endp, 10);
      if (ls.empty() || *endp) die("Line size must be a positive integer.");
      if (file_kt != RMI_KEY_U64) die("Can only construct a bounded RMI on u64 data.");
      auto t0 = std::chrono::steady_clock::now();
      rmi_spline_point* pts = nullptr;
      uint64_t num_pts = 0;
      if (rmi_cache_fix_device(ds, cf.line_size, &pts, &num_pts, nullptr) != RMI_OK) die(rmi_last_error());
      spline.reserve(num_pts);
      for (uint64_t i = 0; i < num_pts; ++i) spline.emplace_back(pts[i].key, pts[i].offset);
      rmi_spline_free(pts);
      std::fprintf(stderr, "Bounded spline compressed data to %.0f%% of original (%zu points, constructed from %llu points).\n",
                   std::round((double)spline.size() / (double)num_rows * 100.0), spline.size(), (unsigned long long)num_rows);
      std::vector<uint64_t> knot_keys(spline.size());
      for (size_t i = 0; i < spline.size(); ++i) knot_keys[i] = spline[i].first;
      rmi_dataset* kds = nullptr;
      if (rmi_dataset_create(knot_keys.data(), knot_keys.size(), RMI_KEY_U64, device, &kds) != RMI_OK) die(rmi_last_error());
      if (rmi_train(kds, a.pos[2].c_str(), std::strtoull(a.pos[3].c_str(), nullptr, 10), flags, &r) != RMI_OK) die(rmi_last_error());
      rmi_dataset_destroy(kds);
      cf.spline = &spline;
      cf.num_data_rows = num_rows;
      bounded = true;
      bounded_build_ns = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    } else {
      if (a.pos.size() < 4) die("called `Option::unwrap()` on a `None` value (models and branching factor are required)");
      train_one(a.pos[2], std::strtoull(a.pos[3].c_str(), nullptr, 10), &r);
    }
    print_stats(*r, num_rows);
    if (!a.has("--no-code")) {
      const uint64_t bt = a.has("--zero-build-time") ? 0 : ((bounded || sized) ? bounded_build_ns : r->build_time_ns);
      try { output_rmi(ns, *r, data_dir, code_kt, !a.has("--no-errors"), bt, ".", bounded ? &cf : nullptr); }
      catch (std::exception& e) { die(e.what()); }
    }
    rmi_result_free(r);
  }
  rmi_dataset_destroy(ds);
  return 0;
}
