// The CPU oracle's error pass over GIVEN tables (rmi_evaluate's reference): train_two_layer's steps after the leaf
// fit (rmi_oracle.cpp, two_layer.rs:178-284) — lower-bound correction, forward pass, widening, statistics — run on a
// table RMI (oracle_tables.cpp) and a key set, WITHOUT the empty-leaf constant replacement (the tables are given,
// not fitted).  The top model must be monotone on the keys, as two_layer.rs:50 asserts during a build.
// The oracle's source is included unchanged.  Built by tests/test_artefacts_host.py with the oracle's flags.
#include "oracle_tables.cpp"

namespace {

template <class T>
Handle* do_evaluate(const TrainedRMI& given, const void* keys, uint64_t n) {
  Data<T> md;
  md.keys = (const T*)keys;
  md.n = (size_t)n;
  REF_ASSERT(n > 0, "start index was 0 but end index was 0");
  const uint64_t num_leaf_models = given.branching_factor;
  const Model& top_model = *given.top;
  auto top_pred = [&](T k) { return top_model.predict_to_int(KeyTraits<T>::to_model_input(k)); };
  {   // two_layer.rs:50 over the whole key set
    uint64_t last_target = 0;
    for (size_t i = 0; i < md.len(); ++i) {
      uint64_t target = std::min<uint64_t>(num_leaf_models - 1, top_pred(md.get_key(i)));
      REF_ASSERT(target >= last_target, "assertion failed: target >= last_target");
      last_target = target;
    }
  }
  const std::vector<Model>& leaf_models = given.leaves;
  const size_t num_rows = md.len();

  LowerBoundCorrection<T> lb(top_pred, num_leaf_models, md);

  std::vector<std::pair<uint64_t, uint64_t>> l1s((size_t)num_leaf_models, {0, 0});
  {
    FixDupsIter<T> it(md);
    T k; size_t y;
    while (it.next(k, y)) {
      ModelInput x = KeyTraits<T>::to_model_input(k);
      uint64_t leaf_idx = top_model.predict_to_int(x);
      size_t target = (size_t)std::min<uint64_t>(num_leaf_models - 1, leaf_idx);
      uint64_t pred = leaf_models[target].predict_to_int(x);
      uint64_t err = error_between(pred, (uint64_t)y, (uint64_t)md.len());
      l1s[target] = {l1s[target].first + 1, std::max(err, l1s[target].second)};
    }
  }
  for (size_t leaf_idx = 0; leaf_idx < (size_t)num_leaf_models; ++leaf_idx) {
    uint64_t curr_err = l1s[leaf_idx].second;
    uint64_t upper_error;
    {
      size_t idx_of_next = lb.next[leaf_idx].first;
      T key_of_next = lb.next[leaf_idx].second;
      uint64_t pred = leaf_models[leaf_idx].predict_to_int(
          KeyTraits<T>::to_model_input(KeyTraits<T>::minus_epsilon(key_of_next)));
      upper_error = error_between(pred, (uint64_t)idx_of_next + 1, (uint64_t)md.len());
    }
    uint64_t lower_error;
    {
      T first_key_before = lb.prev[leaf_idx].second;
      size_t prev_idx = leaf_idx == 0 ? 0 : leaf_idx - 1;
      size_t first_idx = lb.next[prev_idx].first;
      uint64_t pred = leaf_models[leaf_idx].predict_to_int(
          KeyTraits<T>::to_model_input(KeyTraits<T>::plus_epsilon(first_key_before)));
      lower_error = error_between(pred, (uint64_t)first_idx, (uint64_t)md.len());
    }
    uint64_t new_err = std::max(curr_err, std::max(upper_error, lower_error)) + lb.run_lengths[leaf_idx];
    l1s[leaf_idx] = {l1s[leaf_idx].first, new_err};
  }

  auto h = std::make_unique<Handle>();
  TrainedRMI& r = h->rmi;
  {
    size_t m_idx = 0; uint64_t m_err = l1s[0].second;
    for (size_t i = 1; i < l1s.size(); ++i)
      if (l1s[i].second >= m_err) { m_err = l1s[i].second; m_idx = i; }
    r.model_max_error = m_err;
    r.model_max_error_idx = m_idx;
  }
  {
    uint64_t s = 0;
    for (auto& p : l1s) s += p.first * p.second;
    r.model_avg_error = (double)s / (double)num_rows;
  }
  {
    double s = 0.0;
    for (auto& p : l1s) { double v = (double)(p.first * p.second); s += (v * v) / (double)num_rows; }
    r.model_avg_l2_error = s;
  }
  {
    double s = 0.0;
    for (auto& p : l1s) s += (double)p.first * std::log2((double)(2 * p.second + 2));
    r.model_avg_log2_error = s / (double)num_rows;
  }
  r.model_max_log2_error = std::log2((double)r.model_max_error);
  for (auto& p : l1s) { r.leaf_counts.push_back(p.first); r.last_layer_max_l1s.push_back(p.second); }
  r.num_rmi_rows = r.num_data_rows = md.len();
  r.top.reset(new Model(top_model));
  r.leaves = leaf_models;
  r.branching_factor = num_leaf_models;
  return h.release();
}

}  // namespace

extern "C" {

// A new oracle handle: the tables of `tables` (rmi_oracle_from_tables) with errors, counts and statistics measured on
// the n keys.  NULL (rmi_oracle_last_error) where the reference would panic.
void* rmi_oracle_evaluate(void* tables, const void* keys, uint64_t n, int key_type) {
  try {
    g_err.clear();
    const TrainedRMI& given = ((Handle*)tables)->rmi;
    switch (key_type) {
      case 0: return do_evaluate<uint64_t>(given, keys, n);
      case 1: return do_evaluate<uint32_t>(given, keys, n);
      case 2: return do_evaluate<double>(given, keys, n);
      default: g_err = "bad key type"; return nullptr;
    }
  } catch (Panic& p) {
    g_err = p.msg;
    return nullptr;
  }
}

}  // extern "C"
