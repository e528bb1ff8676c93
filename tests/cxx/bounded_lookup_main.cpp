// Evaluates a generated `--bounded` RMI (rmi.h / rmi.cpp from output_rmi with cache-fix knots) on a query file:
//   bounded_lookup <data_dir> <queries: packed u64> <out: packed u64 pos>
// Writes lookup(q, &err) for every query, and fails if err is not the line size given as LINE_SIZE (-D).
#include <cstdint>
#include <cstdio>
#include <vector>
#include "rmi.h"

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  FILE* f = std::fopen(argv[2], "rb");
  if (!f) return 2;
  std::fseek(f, 0, SEEK_END);
  const long bytes = std::ftell(f);
  std::fseek(f, 0, SEEK_SET);
  std::vector<uint64_t> q(bytes / sizeof(uint64_t)), out(q.size());
  if (std::fread(q.data(), sizeof(uint64_t), q.size(), f) != q.size()) return 2;
  std::fclose(f);
  if (!rmi::load(argv[1])) { std::printf("load failed\n"); return 3; }
  for (size_t i = 0; i < q.size(); ++i) {
    size_t err = 0;
    out[i] = rmi::lookup(q[i], &err);
    if (err != LINE_SIZE) { std::printf("err %zu at query %zu\n", err, i); return 1; }
  }
  rmi::cleanup();
  FILE* o = std::fopen(argv[3], "wb");
  if (!o || std::fwrite(out.data(), sizeof(uint64_t), out.size(), o) != out.size()) return 2;
  std::fclose(o);
  return 0;
}
