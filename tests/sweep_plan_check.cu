// Host-only driver of the Karto sweep plan (csrc/karto_sweep_plan.cuh) for tests/test_sweep_plan*.py: no kernel, no
// CUDA call, so it runs on a machine without a GPU.  One request per stdin line, one JSON object per stdout line:
//   layout <search_size> <resolution> <smear_deviation> <range_threshold>
//   plan   <the same four> <n> <batch> <offset_x> <offset_y> <res_x> <res_y> <angle_offset> <angle_res> <fine>
//          <k_first> <na_override> <force_kernel> <sat_valid> <grid_high_bytes> <num_sms> <smem_optin> <win_static>
//                                          -> every SweepPlan field, both pool_layouts and the bound's staged bytes
//   chunks <quantum> <units> <n> <warps> <cap>   -> {"chunks": split_chunks} of the window (4) or the bound (32)
//   ranges <quantum> <total> <chunks>            -> {"ranges": [[lo, hi], ...]} of split_range
//   split  <chunks> <count0> .. <count7>         -> {"items": [[lo, hi, off0, len0, .., off7, len7], ...]}: the
//                                                   window's ranges of its 8 groups, mapped back by chunk_groups
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

static void print_pool(const char *name, const PoolLayout &l) {
  printf(", \"%s\": {\"lead\": %d, \"plane\": %d, \"bytes\": %d, \"pitch\": %zu, \"fits\": %d}", name, l.lead, l.plane,
         l.bytes, l.pitch, (int)l.fits);
}

static int bad(const std::string &line) {
  fprintf(stderr, "bad request: %s\n", line.c_str());
  return 2;
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    if (!(in >> cmd)) continue;
    if (cmd == "chunks") {
      int quantum, units, n, warps, cap;
      if (!(in >> quantum >> units >> n >> warps >> cap) || (quantum != 4 && quantum != 32)) return bad(line);
      printf("{\"chunks\": %d}\n", quantum == 4 ? split_chunks<4, WIN_CHUNK_MIN_BEAMS>(units, n, warps, cap)
                                                 : split_chunks<32, BOUND_CHUNK_MIN_BEAMS>(units, n, warps, cap));
      continue;
    }
    if (cmd == "ranges") {
      int quantum, total, C;
      if (!(in >> quantum >> total >> C) || (quantum != 4 && quantum != 32)) return bad(line);
      printf("{\"ranges\": [");
      for (int c = 0; c < C; c++) {
        int lo, hi;
        if (quantum == 4) split_range<4>(total, c, C, lo, hi);
        else split_range<32>(total, c, C, lo, hi);
        printf("%s[%d, %d]", c ? ", " : "", lo, hi);
      }
      printf("]}\n");
      continue;
    }
    if (cmd == "split") {
      int C;
      int32_t cnt[8];
      if (!(in >> C)) return bad(line);
      for (int g = 0; g < 8; g++)
        if (!(in >> cnt[g])) return bad(line);
      const int total = cnt[0] + cnt[1] + cnt[2] + cnt[3] + cnt[4] + cnt[5] + cnt[6] + cnt[7];
      printf("{\"items\": [");
      for (int c = 0; c < C; c++) {
        int lo, hi, off[8], len[8];
        split_range<4>(total, c, C, lo, hi);
        chunk_groups(cnt, lo, hi, off, len);
        printf("%s[%d, %d", c ? ", " : "", lo, hi);
        for (int g = 0; g < 8; g++) printf(", %d, %d", off[g], len[g]);
        printf("]");
      }
      printf("]}\n");
      continue;
    }
    b2s_matcher_params p = {};
    if (!(in >> p.search_size >> p.resolution >> p.smear_deviation >> p.range_threshold)) return bad(line);
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
    if (cmd != "plan" ||
        !(in >> n >> batch >> s.offset_x >> s.offset_y >> s.res_x >> s.res_y >> s.angle_offset >> s.angle_res >>
          s.fine >> k_first >> na_override >> force_kernel >> sat_valid >> grid_high_bytes >> num_sms >> smem_optin >>
          win_static))
      return bad(line);
    const int sbx = (g.width_step + 3) / 4, sby = (g.height + 3) / 4;  // as b2s_matcher_create sets them
    const SweepPlan pl = plan_sweep(p, g, s, n, batch, k_first, na_override, force_kernel, sat_valid != 0,
                                    grid_high_bytes != 0, sbx, sby, num_sms, smem_optin, win_static);
    printf("{");
    print_grid(g);
    print_pool("pool", pool_layout(g, 4, smem_optin, win_static));
    print_pool("pool7", pool_layout(g, 7, smem_optin, win_static));
    printf(", \"stage\": %zu, \"stage7\": %zu, \"sat_bytes\": %zu", bound_stage_bytes(n, pl.skip_empty, sbx, sby),
           bound_stage_bytes(n, false, sbx, sby), sizeof(uint16_t) * sat_stride(sbx, sby));
    printf(", \"status\": %d, \"error\": \"%s\"", (int)pl.status, pl.error ? pl.error : "");
    if (!pl.status)
      printf(", \"nx\": %d, \"ny\": %d, \"na\": %d, \"stride\": %d, \"use_window\": %d, \"need_plain_lut\": %d, "
             "\"copy_bytes\": %d, \"tiles_x\": %d, \"tiles_y\": %d, \"rows_total\": %d, \"halo_rows\": %d, "
             "\"band_rows\": %d, \"nbands\": %d, \"band_bytes\": %d, \"neg_bands\": %d, \"win_smem\": %zu, \"gen\": %d, "
             "\"ctas\": %d, \"skip_empty\": %d, \"osm\": %zu, \"prune\": %d, \"bound_stage\": %d, \"bound_smem\": %zu, "
             "\"group\": %d, \"group_stage\": %d, \"group_smem\": %zu, \"bound_rows\": %d, \"group_rows\": %d, "
             "\"acc_slots\": %d, \"listed_smem\": %zu",
             pl.nx, pl.ny, pl.na, pl.stride, (int)pl.use_window, (int)pl.need_plain_lut, pl.copy_bytes, pl.tiles_x,
             pl.tiles_y, pl.rows_total, pl.halo_rows, pl.band_rows, pl.nbands, pl.band_bytes, pl.neg_bands, pl.win_smem,
             (int)pl.gen, pl.ctas, (int)pl.skip_empty, pl.osm, (int)pl.prune, (int)pl.bound_stage, pl.bound_smem,
             (int)pl.group, (int)pl.group_stage, pl.group_smem, pl.bound_rows, pl.group_rows, pl.acc_slots,
             pl.listed_smem);
    printf("}\n");
  }
  return 0;
}
