// GPU harness for tests/test_covisibility.py: cvb_covisibility with its pair budget as an argument.  The budget is an
// argument of the library's internal function (covins_b200/csrc/map_graph.cu, compiled into this translation unit with
// ctx.cu), not a public option: a small budget makes a small map take the chunked path a very large map takes.
//   usage: covis_harness <dir> <K> <min_weight> <pair_budget>
// reads <dir>/ptr.bin (int32 [L+1]), kf.bin (int32 [n_obs]) and, when present, skip.bin (uint8 [n_obs]) and valid.bin
// (uint8 [L]); writes out_ptr.bin, out_kf.bin, out_w.bin (int32) and out_launches.bin (int64: the call's kernel launches).
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "../../covins_b200/csrc/ctx.cu"
#include "../../covins_b200/csrc/map_graph.cu"

template <class V>
static std::vector<V> load(const std::string& path, bool* found = nullptr) {
  std::vector<V> v;
  FILE* f = fopen(path.c_str(), "rb");
  if (found) *found = f != nullptr;
  if (!f) return v;
  fseek(f, 0, SEEK_END);
  const long nb = ftell(f);
  fseek(f, 0, SEEK_SET);
  v.resize((size_t)nb / sizeof(V));
  if (nb && fread(v.data(), 1, (size_t)nb, f) != (size_t)nb) exit(2);
  fclose(f);
  return v;
}
static void store(const std::string& path, const void* p, size_t bytes) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f || (bytes && fwrite(p, 1, bytes, f) != bytes)) exit(2);
  fclose(f);
}

int main(int argc, char** argv) {
  if (argc != 5) return 2;
  const std::string dir = argv[1];
  const int K = atoi(argv[2]), min_weight = atoi(argv[3]);
  const int64_t budget = atoll(argv[4]);
  bool has_skip = false, has_valid = false;
  const auto ptr = load<int32_t>(dir + "/ptr.bin");
  const auto kf = load<int32_t>(dir + "/kf.bin");
  const auto skip = load<uint8_t>(dir + "/skip.bin", &has_skip);
  const auto valid = load<uint8_t>(dir + "/valid.bin", &has_valid);
  if (ptr.empty()) return 2;
  cvb_ctx* ctx = nullptr;
  if (cvb_ctx_create(0, &ctx) != CVB_OK) {
    fprintf(stderr, "no CUDA device\n");
    return 3;
  }
  std::vector<int32_t> nbr_ptr((size_t)K + 1), nbr_kf, nbr_w;
  int64_t n_total = 0, cap = 0;
  for (int call = 0; call < 2; call++) {   // size, then fill
    nbr_kf.resize((size_t)cap + 1);
    nbr_w.resize((size_t)cap + 1);
    const int64_t before = cvb_launch_count(ctx);
    const int rc = cvb_covisibility_budgeted(ctx, K, (int)ptr.size() - 1, ptr.data(), kf.data(), has_skip ? skip.data() : nullptr,
                                             has_valid ? valid.data() : nullptr, min_weight, nbr_ptr.data(), nbr_kf.data(), nbr_w.data(), cap,
                                             &n_total, budget);
    if (rc != CVB_OK) {
      fprintf(stderr, "status %d: %s\n", rc, cvb_last_error(ctx));
      return 4;
    }
    const int64_t launches = cvb_launch_count(ctx) - before;
    store(dir + "/out_launches.bin", &launches, sizeof launches);
    cap = n_total;
  }
  store(dir + "/out_ptr.bin", nbr_ptr.data(), nbr_ptr.size() * sizeof(int32_t));
  store(dir + "/out_kf.bin", nbr_kf.data(), (size_t)n_total * sizeof(int32_t));
  store(dir + "/out_w.bin", nbr_w.data(), (size_t)n_total * sizeof(int32_t));
  cvb_ctx_destroy(ctx);
  return 0;
}
