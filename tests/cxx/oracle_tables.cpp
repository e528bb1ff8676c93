// The CPU oracle's lookup (rmi_oracle_lookup, codegen.rs:612-718) on GIVEN tables: a top model and N leaf
// parameter rows plus error bounds, e.g. the ones the GPU trained.  A GPU-vs-oracle lookup comparison then checks
// the evaluation alone, bit for bit, whatever tolerance the training of a model is held to.  The oracle's source
// is included unchanged, so the models are evaluated by exactly the code the oracle trains with.
// Built by tests/lookup_oracle.py with the oracle's compiler flags.
#include "../../oracle/rmi_oracle.cpp"

extern "C" {

// top: kind (rmi_model_id), bradix high, radix table bits, float / integer parameters in Model::params() order,
// radix hint table (t32), histogram radix index (a1) and pivots (a2).  leaves: N x ppm parameters and N error
// bounds of kind leaf_kind.  n: number of keys the RMI was trained on.  Returns NULL (rmi_oracle_last_error) on a
// malformed description.
void* rmi_oracle_from_tables(int top_kind, int high, int table_bits, const double* fp, int nfp, const uint64_t* ip,
                             int nip, const uint32_t* t32, uint64_t t32_len, const uint64_t* a1, uint64_t a1_len,
                             const uint64_t* a2, uint64_t a2_len, int leaf_kind, const double* params, int ppm,
                             const uint64_t* errors, uint64_t N, uint64_t n) {
  g_err.clear();
  if (top_kind < K_LINEAR || top_kind > K_HISTOGRAM || leaf_kind < K_LINEAR || leaf_kind > K_LOGNORMAL || N == 0 ||
      n == 0 || (ppm && !params) || !errors) {
    g_err = "rmi_oracle_from_tables: bad argument";
    return nullptr;
  }
  auto h = std::make_unique<Handle>();
  TrainedRMI& r = h->rmi;
  Model top((Kind)top_kind);
  top.fp.assign(fp, fp + nfp);
  top.ip.assign(ip, ip + nip);
  if (t32) top.t32.assign(t32, t32 + t32_len);
  if (a1) top.a1.assign(a1, a1 + a1_len);
  if (a2) top.a2.assign(a2, a2 + a2_len);
  top.high = high != 0;
  top.table_bits = (uint8_t)table_bits;
  r.top.reset(new Model(std::move(top)));
  r.leaves.reserve((size_t)N);
  for (uint64_t j = 0; j < N; ++j) {
    Model m((Kind)leaf_kind);
    m.fp.assign(params + j * (uint64_t)ppm, params + (j + 1) * (uint64_t)ppm);
    r.leaves.push_back(std::move(m));
  }
  r.last_layer_max_l1s.assign(errors, errors + N);
  r.leaf_counts.assign((size_t)N, 0);
  r.branching_factor = N;
  r.num_rmi_rows = r.num_data_rows = n;
  return h.release();
}

}  // extern "C"
