// Host-only harness for tests/test_tile_levels.py: builds a cvb_chol::TilePlan from a tile mask and writes its level data.
// Input: as tests/cpp/tile_plan_dump.cu (int32: nt, has_group, has_owner, rank, mask[nt * nt], col_group[nt]?, owner[nt]?).
// Output (int32, binary): sections [length, values...]: col_ptr, row_idx, pair_ptr, pair_i, pair_j, pair_mask, pair_k0,
// lvl_ptr, lvl_pair_ptr, lvl_pair_i, lvl_pair_j, lvl_pair_k0, lvl_pair_mask, lvl_trsm_ptr, lvl_trsm_tile, lvl_trsm_col,
// lvl_fwd_ptr, lvl_fwd_idx, lvl_bwd_ptr, lvl_bwd_idx, col_base, rowc_ptr, rowc_idx.
//   tile_plan_levels_dump layout in.bin out.bin: the column groups' tile layout (cvb_chol::nd_layout).  Input (int32): bw,
//   n_groups, sizes[n_groups] (group g's blocks are the next sizes[g] block ids).  Output: off[blocks], group_of_tile[].
// Needs no GPU: TilePlan::build and nd_layout are host code and nothing here calls the CUDA runtime.
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../covins_b200/csrc/cholesky.cuh"

// the library's error helper (referenced by cholesky.cu's device paths, never called here)
int cvb_fail(cvb_ctx*, int code, const char*, ...) { return code; }

static void put(FILE* f, const std::vector<int>& v) {
  const int32_t n = (int32_t)v.size();
  fwrite(&n, 4, 1, f);
  if (n) fwrite(v.data(), 4, v.size(), f);
}

static int layout(const char* in, const char* out) {
  FILE* f = fopen(in, "rb");
  if (!f) return 2;
  int32_t hdr[2];
  if (fread(hdr, 4, 2, f) != 2 || hdr[0] < 1 || hdr[0] > cvb_chol::T || hdr[1] < 0) return 2;
  std::vector<int32_t> sizes(hdr[1]);
  if (fread(sizes.data(), 4, sizes.size(), f) != sizes.size()) return 2;
  fclose(f);
  std::vector<std::vector<int>> members(sizes.size());
  int next = 0;
  for (size_t g = 0; g < sizes.size(); g++)
    for (int q = 0; q < sizes[g]; q++) members[g].push_back(next++);
  std::vector<int> off(next, -1), group_of_tile;
  cvb_chol::nd_layout(members, hdr[0], off, group_of_tile);
  f = fopen(out, "wb");
  if (!f) return 2;
  put(f, off);
  put(f, group_of_tile);
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 4 && std::string(argv[1]) == "layout") return layout(argv[2], argv[3]);
  if (argc != 3) {
    fprintf(stderr, "usage: %s [layout] in.bin out.bin\n", argv[0]);
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
  cvb_chol::TilePlan p;
  p.build(nt, mask, std::vector<int>(group.begin(), group.end()), hdr[2] ? &owner : nullptr, hdr[3]);
  f = fopen(argv[2], "wb");
  if (!f) return 2;
  for (const std::vector<int>* v :
       {&p.h_col_ptr, &p.h_row_idx, &p.h_pair_ptr, &p.h_pair_i, &p.h_pair_j, &p.h_pair_mask, &p.h_pair_k0, &p.h_lvl_ptr,
        &p.h_lvl_pair_ptr, &p.h_lvl_pair_i, &p.h_lvl_pair_j, &p.h_lvl_pair_k0, &p.h_lvl_pair_mask, &p.h_lvl_trsm_ptr,
        &p.h_lvl_trsm_tile, &p.h_lvl_trsm_col, &p.h_lvl_fwd_ptr, &p.h_lvl_fwd_idx, &p.h_lvl_bwd_ptr, &p.h_lvl_bwd_idx,
        &p.h_col_base, &p.h_rowc_ptr, &p.h_rowc_idx})
    put(f, *v);
  fclose(f);
  return 0;
}
