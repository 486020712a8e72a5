// Host-only harness for tests/test_tile_plan.py: builds a cvb_chol::TilePlan from a tile mask and writes its launch lists.
// Input (int32, binary): nt, has_group, has_owner, rank, mask[nt * nt] (lower, row-major), col_group[nt]?, owner[nt]?
// Output (int32, binary): a sequence of sections [length, values...]: col_ptr, row_idx, pair_ptr, pair_i, pair_j, pair_mask,
// pair_k0, pair_split, blk_end, {kPanelBlock}, {flops / (2 * 128^3)}.
// Needs no GPU: TilePlan::build is host code and nothing here calls the CUDA runtime.
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../covins_b200/csrc/cholesky.cuh"

// the library's error helper (referenced by cholesky.cu's device paths, never called here)
int cvb_fail(cvb_ctx*, int code, const char*, ...) { return code; }

static void put(FILE* f, const std::vector<int>& v) {
  const int32_t n = (int32_t)v.size();
  fwrite(&n, 4, 1, f);
  if (n) fwrite(v.data(), 4, v.size(), f);
}

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]);
    return 2;
  }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int32_t hdr[4];
  if (fread(hdr, 4, 4, f) != 4) return 2;
  const int nt = hdr[0];
  std::vector<int32_t> m((size_t)nt * nt), group, owner;
  if (fread(m.data(), 4, m.size(), f) != m.size()) return 2;
  if (hdr[1]) {
    group.resize(nt);
    if (fread(group.data(), 4, nt, f) != (size_t)nt) return 2;
  }
  if (hdr[2]) {
    owner.resize(nt);
    if (fread(owner.data(), 4, nt, f) != (size_t)nt) return 2;
  }
  fclose(f);
  std::vector<uint8_t> mask(m.begin(), m.end());
  cvb_chol::TilePlan plan;
  plan.build(nt, mask, std::vector<int>(group.begin(), group.end()), hdr[2] ? &owner : nullptr, hdr[3]);
  f = fopen(argv[2], "wb");
  if (!f) return 2;
  for (const std::vector<int>* v : {&plan.h_col_ptr, &plan.h_row_idx, &plan.h_pair_ptr, &plan.h_pair_i, &plan.h_pair_j,
                                    &plan.h_pair_mask, &plan.h_pair_k0, &plan.h_pair_split, &plan.h_blk_end})
    put(f, *v);
  put(f, {cvb_chol::kPanelBlock});
  put(f, {(int)(plan.flops / (2.0 * cvb_chol::T * cvb_chol::T * cvb_chol::T) + 0.5)});
  fclose(f);
  return 0;
}
