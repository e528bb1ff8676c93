// optimizer.hpp — the reference's two-phase configuration search (rmi_lib/src/optimizer.rs),
// CPU-side: the search loop stays on the host, every candidate is a statistics-only build
// (only avg/max log2 error and the model size are consumed, optimizer.rs:163-171), so no leaf
// table ever leaves the GPU during a sweep.  How a group of candidates is measured is a
// parameter (MeasureStep): replicas of the whole key set, or range-partitioned slabs.
#pragma once
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <set>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../include/rmi_b200.h"
#include "codegen.hpp"

namespace rmihost {

struct RMIStatistics {   // optimizer.rs:153-160
  std::string models;
  uint64_t branching_factor = 0;
  double average_log2_error = 0, max_log2_error = 0;
  uint64_t size = 0;

  bool dominated_by(const RMIStatistics& o) const {   // :173-187
    if (size < o.size) return false;
    if (average_log2_error < o.average_log2_error) return false;
    if (size == o.size && average_log2_error <= o.average_log2_error) return false;
    double d = std::fabs(average_log2_error - o.average_log2_error);
    if (size <= o.size && d < 2.220446049250313e-16) return false;
    return true;
  }
  bool has_config(const std::string& m, uint64_t bf) const { return models == m && branching_factor == bf; }
};

inline std::string optimizer_profile() {
  const char* p = std::getenv("RMI_OPTIMIZER_PROFILE");
  std::string s = p ? p : "";
  if (!s.empty() && s != "fast" && s != "memory" && s != "disk") throw std::runtime_error("Invalid optimizer profile " + s);
  return s;
}
inline std::vector<std::string> top_only_layers() {   // :15-28
  std::string p = optimizer_profile();
  if (p == "fast") return {"robust_linear"};
  if (p == "disk") return {"radix", "radix18", "radix22", "robust_linear", "normal", "lognormal", "loglinear"};
  return {"radix", "radix18", "radix22", "robust_linear"};
}
inline std::vector<std::string> anywhere_layers() {   // :30-41
  if (optimizer_profile() == "fast") return {"linear", "cubic"};
  return {"linear", "cubic", "linear_spline"};
}
inline std::vector<uint64_t> branching_factors() {   // :43-57
  std::string p = optimizer_profile();
  int hi = p == "disk" ? 28 : 25, step = p == "fast" ? 2 : 1;
  std::vector<uint64_t> v;
  for (int i = 6; i < hi; i += step) v.push_back((uint64_t)1 << i);
  return v;
}

inline std::vector<RMIStatistics> pareto_front(const std::vector<RMIStatistics>& r) {   // :59-72
  std::vector<RMIStatistics> front;
  for (auto& x : r) {
    bool dominated = false;
    for (auto& v : r) if (x.dominated_by(v)) { dominated = true; break; }
    if (!dominated) front.push_back(x);
  }
  return front;
}

inline std::vector<RMIStatistics> narrow_front(const std::vector<RMIStatistics>& results, size_t desired) {   // :74-108
  if (desired < 2) throw std::runtime_error("assertion failed: desired_size >= 2");
  if (results.size() <= desired) return results;
  std::vector<RMIStatistics> tmp = results;
  std::stable_sort(tmp.begin(), tmp.end(), [](const RMIStatistics& a, const RMIStatistics& b) { return a.size < b.size; });
  RMIStatistics best = tmp.front();
  tmp.erase(tmp.begin());
  while (tmp.size() > desired - 1) {
    size_t gi = 0;
    double gv = 0;
    bool have = false;
    for (size_t i = 0; i + 1 < tmp.size(); ++i) {   // min_by keeps the first minimum
      double v = (double)tmp[i + 1].size / (double)tmp[i].size;
      if (!have || v < gv) { gv = v; gi = i; have = true; }
    }
    double e1 = tmp[gi].average_log2_error, e2 = tmp[gi + 1].average_log2_error;
    if (e1 > e2) tmp.erase(tmp.begin() + gi); else tmp.erase(tmp.begin() + gi + 1);
  }
  tmp.insert(tmp.begin(), best);
  return tmp;
}

typedef std::pair<std::string, uint64_t> Config;

inline std::vector<Config> first_phase_configs() {   // :110-125
  std::vector<Config> out;
  std::vector<std::string> tops = top_only_layers();
  for (auto& a : anywhere_layers()) tops.push_back(a);
  auto bfs = branching_factors();
  for (auto& t : tops)
    for (auto& b : anywhere_layers())
      for (size_t i = 0; i < bfs.size(); i += 5) out.push_back({t + "," + b, bfs[i]});
  return out;
}
inline std::vector<Config> second_phase_configs(const std::vector<RMIStatistics>& first) {   // :127-151
  std::set<std::string> qualifying;   // BTreeSet: sorted iteration
  for (auto& r : pareto_front(first)) qualifying.insert(r.models);
  std::vector<Config> out;
  for (auto& m : qualifying)
    for (uint64_t bf : branching_factors()) {
      bool seen = false;
      for (auto& v : first) if (v.has_config(m, bf)) { seen = true; break; }
      if (!seen) out.push_back({m, bf});
    }
  return out;
}

// measure_rmis (:220-231).  The unit of measurement is a GROUP: the configurations "top,leaves[k]" that share a top
// model and a branching factor.  A MeasureStep measures one group and returns its K statistics (average / max log2
// error and size, in leaves[] order; models and branching factor are filled in here); it throws std::runtime_error
// to abort the sweep, as a panicking configuration aborts the reference's.  Groups keep the order of their first
// member and are measured longest first (smallest branching factor first: the smaller the branching factor, the longer
// the per-lane chains); results land at the configurations' own positions.  `workers` host threads pull the next
// group from a shared counter; the step learns which thread calls it.  Two steps exist: the replicas' (below) and a
// caller's C callback (rmi_find_pareto_efficient_configs_with, used for range-partitioned keys).
struct MeasureGroup {
  std::string top;                  // the bare top-model name, or (batched == false) the whole model spec
  uint64_t bf = 0;
  std::vector<std::string> leaves;  // batched == false: one entry
  std::vector<size_t> index;        // positions of the configurations
  bool batched = true;
};
struct MeasureStep {
  std::function<std::vector<RMIStatistics>(size_t worker, const MeasureGroup& g)> measure;
  size_t workers = 1;
  // Keep a configuration apart when true (small branching factors when batching is on): the replicas balance them.
  std::function<bool(const std::string& top, const std::string& leaf, uint64_t bf)> keep_apart;
};

inline std::vector<RMIStatistics> measure_rmis(const MeasureStep& step, const std::vector<Config>& configs) {
  std::vector<RMIStatistics> out(configs.size());
  std::vector<MeasureGroup> groups;
  for (size_t i = 0; i < configs.size(); ++i) {
    const std::string& m = configs[i].first;
    const size_t comma = m.find(',');
    const std::string top = m.substr(0, comma), leaf = comma == std::string::npos ? "" : m.substr(comma + 1);
    const bool batchable = comma != std::string::npos && leaf.find(',') == std::string::npos &&
                           !(step.keep_apart && step.keep_apart(top, leaf, configs[i].second));
    MeasureGroup* g = nullptr;
    if (batchable)
      for (auto& c : groups) if (c.batched && c.top == top && c.bf == configs[i].second) { g = &c; break; }
    if (!g) {
      groups.push_back(MeasureGroup{batchable ? top : m, configs[i].second, {}, {}, batchable});
      g = &groups.back();
    }
    g->leaves.push_back(leaf);
    g->index.push_back(i);
  }
  std::vector<size_t> order(groups.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return groups[a].bf < groups[b].bf; });
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  const size_t W = std::max<size_t>(1, step.workers);
  std::vector<std::string> errors(W);
  auto worker = [&](size_t w) {
    for (;;) {
      size_t oi = next.fetch_add(1);
      if (oi >= groups.size() || failed.load()) return;
      const MeasureGroup& g = groups[order[oi]];
      std::vector<RMIStatistics> res;
      try {
        res = step.measure(w, g);
        if (res.size() != g.index.size()) throw std::runtime_error("the measuring step returned " + std::to_string(res.size()) +
                                                                   " results for " + std::to_string(g.index.size()) + " configurations");
      } catch (const std::exception& e) {
        errors[w] = "training " + configs[g.index[0]].first + " " + std::to_string(g.bf) + ": " + e.what();
        failed.store(true);
        return;
      }
      for (size_t k = 0; k < g.index.size(); ++k) {
        const Config& c = configs[g.index[k]];
        RMIStatistics& s = out[g.index[k]];
        s = res[k];
        s.models = c.first; s.branching_factor = c.second;
      }
    }
  };
  if (W == 1) worker(0);
  else {
    std::vector<std::thread> th;
    for (size_t w = 0; w < W; ++w) th.emplace_back([&worker, w] { worker(w); rmi_thread_release(); });
    for (auto& t : th) t.join();
  }
  for (auto& e : errors) if (!e.empty()) throw std::runtime_error(e);
  return out;
}

// The replicas' step: `replicas` holds the SAME key set on one or more devices (rmi_dataset_replicate), one host thread
// per replica.  The reference maps the configurations over a rayon pool on one shared data set (optimizer.rs:224-229);
// here every configuration is an independent stats-only build, with no communication.  A batched group is one
// rmi_train_stats_batch (one top fit and one boundary pass for the whole group, SURVEY.md section 8(f)2).  Batching pays
// where the shared passes are a visible part of a configuration's cost: at small branching factors a configuration's
// time is its leaves' serial recurrences (n / bf keys per lane), and keeping such configurations apart lets the replicas
// balance them.  RMI_OPTIMIZER_NO_BATCH=1 measures every configuration on its own.
inline MeasureStep replica_step(const std::vector<const rmi_dataset*>& replicas, uint32_t flags, bool verbose) {
  static const bool batching = [] { const char* e = std::getenv("RMI_OPTIMIZER_NO_BATCH"); return !(e && e[0] == '1'); }();
  MeasureStep s;
  s.workers = replicas.size();
  s.keep_apart = [](const std::string&, const std::string&, uint64_t bf) { return !batching || bf < 4096; };
  s.measure = [replicas, flags, verbose](size_t w, const MeasureGroup& g) {
    const rmi_dataset* ds = replicas[w];
    const size_t K = g.index.size();
    std::vector<rmi_result*> res(K, nullptr);
    int rc;
    if (g.batched) {   // g.top holds the bare top-model name
      std::vector<const char*> names;
      for (auto& l : g.leaves) names.push_back(l.c_str());
      rc = rmi_train_stats_batch(ds, g.top.c_str(), names.data(), (int)K, g.bf, flags, res.data());
    } else {
      rc = rmi_train(ds, g.top.c_str(), g.bf, flags | RMI_FLAG_STATS_ONLY, &res[0]);
    }
    if (rc != RMI_OK) throw std::runtime_error(rmi_last_error());
    std::vector<RMIStatistics> out(K);
    for (size_t k = 0; k < K; ++k) {
      rmi_result* r = res[k];
      out[k].average_log2_error = r->model_avg_log2_error; out[k].max_log2_error = r->model_max_log2_error;
      out[k].size = rmi_size(*r, true);
      if (verbose) std::fprintf(stderr, "  [replica %zu] %-28s %10llu  avg_log2 %.5f  size %llu  (%.2f ms)\n", w,
                                (g.batched ? g.top + "," + g.leaves[k] : g.top).c_str(), (unsigned long long)g.bf,
                                out[k].average_log2_error, (unsigned long long)out[k].size, r->device_time_ns / 1e6);
      rmi_result_free(r);
    }
    return out;
  };
  return s;
}

inline std::vector<RMIStatistics> find_pareto_efficient_configs(const MeasureStep& step, size_t restrict_to) {   // :233-249
  auto first = measure_rmis(step, first_phase_configs());
  auto second = measure_rmis(step, second_phase_configs(first));
  auto front = narrow_front(pareto_front(second), restrict_to);
  std::stable_sort(front.begin(), front.end(),
                   [](const RMIStatistics& a, const RMIStatistics& b) { return a.average_log2_error < b.average_log2_error; });
  return front;
}

inline std::vector<RMIStatistics> find_pareto_efficient_configs(const std::vector<const rmi_dataset*>& replicas, size_t restrict_to,
                                                                uint32_t flags, bool verbose) {
  return find_pareto_efficient_configs(replica_step(replicas, flags, verbose), restrict_to);
}

inline std::vector<RMIStatistics> find_pareto_efficient_configs(const rmi_dataset* ds, size_t restrict_to, uint32_t flags,
                                                                bool verbose) {
  return find_pareto_efficient_configs(std::vector<const rmi_dataset*>{ds}, restrict_to, flags, verbose);
}

inline void display_table(const std::vector<RMIStatistics>& items) {   // :193-206
  std::vector<std::vector<std::string>> rows;
  rows.push_back({"Models", "Branch", "   AvgLg2", "   MaxLg2", "   Size (b)"});
  char buf[64];
  for (auto& it : items) {
    std::vector<std::string> r;
    r.push_back(it.models);
    std::snprintf(buf, sizeof buf, "%10llu", (unsigned long long)it.branching_factor); r.push_back(buf);
    std::snprintf(buf, sizeof buf, "     %.5f", it.average_log2_error); r.push_back(buf);
    std::snprintf(buf, sizeof buf, "     %.5f", it.max_log2_error); r.push_back(buf);
    r.push_back("     " + std::to_string(it.size));
    rows.push_back(r);
  }
  size_t w[5] = {0, 0, 0, 0, 0};
  for (auto& r : rows) for (int c = 0; c < 5; ++c) w[c] = std::max(w[c], r[c].size());
  for (auto& r : rows) {
    std::string line = r[0] + std::string(w[0] - r[0].size(), ' ');
    for (int c = 1; c < 5; ++c) line += " " + std::string(w[c] - r[c].size(), ' ') + r[c];
    std::printf("%s\n", line.c_str());
  }
}

}  // namespace rmihost
