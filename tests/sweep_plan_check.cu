// Host-only driver of the Karto sweep plan (csrc/karto_sweep_plan.cuh) for tests/test_sweep_plan.py: no kernel, no CUDA
// call, so it runs on a machine without a GPU.  One request per stdin line, one JSON object per stdout line:
//   layout <search_size> <resolution> <smear_deviation> <range_threshold>
//   plan   <the same four> <n> <batch> <offset_x> <offset_y> <res_x> <res_y> <angle_offset> <angle_res> <fine>
//          <k_first> <na_override> <force_kernel> <sat_valid> <grid_high_bytes> <num_sms> <smem_optin> <win_static>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/karto_sweep_plan.cuh"

using namespace b2s;

static void print_grid(const b2s_grid_info &g) {
  printf("\"width\": %d, \"height\": %d, \"width_step\": %d, \"data_size\": %d, \"search_side\": %d", g.width, g.height,
         g.width_step, g.data_size, g.search_side);
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    b2s_matcher_params p = {};
    if (!(in >> cmd >> p.search_size >> p.resolution >> p.smear_deviation >> p.range_threshold)) continue;
    const b2s_grid_info g = grid_layout(p);
    if (cmd == "layout") {
      printf("{");
      print_grid(g);
      printf("}\n");
      continue;
    }
    b2s_search s = {};
    int n, batch, k_first, na_override, force_kernel, sat_valid, grid_high_bytes, num_sms, smem_optin;
    size_t win_static;
    if (!(in >> n >> batch >> s.offset_x >> s.offset_y >> s.res_x >> s.res_y >> s.angle_offset >> s.angle_res >>
          s.fine >> k_first >> na_override >> force_kernel >> sat_valid >> grid_high_bytes >> num_sms >> smem_optin >>
          win_static)) {
      fprintf(stderr, "bad request: %s\n", line.c_str());
      return 2;
    }
    const int sbx = (g.width_step + 3) / 4, sby = (g.height + 3) / 4;  // as b2s_matcher_create sets them
    const SweepPlan pl = plan_sweep(p, g, s, n, batch, k_first, na_override, force_kernel, sat_valid != 0,
                                    grid_high_bytes != 0, sbx, sby, num_sms, smem_optin, win_static);
    printf("{");
    print_grid(g);
    printf(", \"status\": %d, \"error\": \"%s\"", (int)pl.status, pl.error ? pl.error : "");
    if (!pl.status)
      printf(", \"nx\": %d, \"ny\": %d, \"na\": %d, \"stride\": %d, \"use_window\": %d, \"need_plain_lut\": %d, "
             "\"copy_bytes\": %d, \"tiles_x\": %d, \"tiles_y\": %d, \"rows_total\": %d, \"halo_rows\": %d, "
             "\"band_rows\": %d, \"nbands\": %d, \"band_bytes\": %d, \"neg_bands\": %d, \"win_smem\": %zu, \"gen\": %d, "
             "\"ctas\": %d, \"skip_empty\": %d, \"osm\": %zu",
             pl.nx, pl.ny, pl.na, pl.stride, (int)pl.use_window, (int)pl.need_plain_lut, pl.copy_bytes, pl.tiles_x,
             pl.tiles_y, pl.rows_total, pl.halo_rows, pl.band_rows, pl.nbands, pl.band_bytes, pl.neg_bands, pl.win_smem,
             (int)pl.gen, pl.ctas, (int)pl.skip_empty, pl.osm);
    printf("}\n");
  }
  return 0;
}
