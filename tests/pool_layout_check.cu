// Host-only check of the bound pass's pooled-image layouts (csrc/karto_sweep_plan.cuh: pool_layout, pool_index) for
// tests/test_pool_layout.py: no kernel, no CUDA call, so it runs without a GPU.  One request per stdin line,
// `<search_size> <resolution> <smear_deviation> <range_threshold> <seed> [K]` (K = 4, the default, or 7), one JSON
// object per stdout line.  For the handle's grid geometry and a seeded grid of bytes 0..127 it builds the staged K x K image as
// k_grid_pool writes it (plane r byte m = P[4m + r - lead], with P restated from its definition) between the kernel's
// WIN_GUARD zero guards and checks:
//   - pool_index maps every f in [-lead, data_size) into its own plane, to a byte no other f takes, holding P[f];
//   - every byte of a plane past the last P[f] with f < data_size is zero;
//   - K = 4 only, as that read is the single-angle pass's: for every interior window origin (win_origin_class: the
//     window of a 32 x 32 tile lies within WIN_GUARD - 16 bytes of the grid) and every block row, k_sweep_bound's
//     three-word read starts at or after the image's first guard byte, ends inside its own plane (or the last guard),
//     and the 8 bytes it keeps are P at the 8 corners.
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/karto_sweep_plan.cuh"

using namespace b2s;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    b2s_matcher_params p = {};
    int K;
    unsigned seed = 0;
    if (!(in >> p.search_size >> p.resolution >> p.smear_deviation >> p.range_threshold >> seed)) continue;
    if (!(in >> K)) K = 4;
    const b2s_grid_info g = grid_layout(p);
    const PoolLayout l = pool_layout(g, K, 232448, 3200);
    const int ws = g.width_step, ds = g.data_size, lead = l.lead, plane = l.plane, bytes = l.bytes;
    std::vector<uint8_t> grid(ds);
    uint32_t s = seed * 2654435761u + 1u;
    for (auto &v : grid) {
      s = s * 1664525u + 1013904223u;
      v = (s >> 24) < 96 ? 0 : (uint8_t)((s >> 8) % 128);
    }
    // P[f] for f in [lo_f, hi_f): wide enough for every corner and every byte the image holds
    const int lo_f = -lead - 4 * WIN_GUARD, hi_f = ds + 4 * WIN_GUARD + 4 * plane;
    std::vector<uint8_t> P(hi_f - lo_f);
    for (int f = lo_f; f < hi_f; f++) {
      int m = 0;
      for (int dy = 0; dy < K; dy++)
        for (int dx = 0; dx < K; dx++) {
          const long long r = (long long)f + dy * ws + dx;
          if (r >= 0 && r < ds) m = grid[r] > m ? grid[r] : m;
        }
      P[f - lo_f] = (uint8_t)m;
    }
    auto Pf = [&](long long f) { return (f < lo_f || f >= hi_f) ? -1 : (int)P[f - lo_f]; };
    std::vector<uint8_t> img(WIN_GUARD + bytes + WIN_GUARD, 0);
    for (int r = 0; r < 4; r++)
      for (int m = 0; m < plane; m++) img[WIN_GUARD + r * plane + m] = (uint8_t)Pf(4LL * m + r - lead);
    std::string err;
    auto fail = [&](const char *what, long long v) {
      if (err.empty()) {
        char b[160];
        snprintf(b, sizeof b, "%s at %lld", what, v);
        err = b;
      }
    };
    std::vector<uint8_t> taken(bytes, 0);
    for (int f = -lead; f < ds && err.empty(); f++) {
      const int i = pool_index(f, lead, plane), r = (f + lead) & 3;
      if (i < r * plane || i >= (r + 1) * plane) fail("pool_index outside the plane of f", f);
      else if (taken[i]++) fail("pool_index not one-to-one", f);
      else if (img[WIN_GUARD + i] != Pf(f)) fail("staged byte is not P[f]", f);
    }
    for (int i = 0; i < bytes && err.empty(); i++)
      if (!taken[i] && img[WIN_GUARD + i] != 0) fail("padding byte is not zero", i);
    const int span = 31 * ws + 32 + 8;  // win_geom's span of a 32 x 32 stride-1 tile
    long long interior = 0;
    int max_end = -1;  // the furthest byte past its plane's start that a read of plane 0..3 reaches, in plane bytes
    for (int a = -(WIN_GUARD - 16) + 8; K == 4 && a + span <= ds + (WIN_GUARD - 16) && err.empty(); a++) {
      interior++;
      const int addr = pool_index(a, lead, plane), r = (a + lead) & 3;
      for (int by = 0; by < 8 && err.empty(); by++) {
        const int b0 = addr + by * ws, wa = b0 & ~3;
        if (wa < -WIN_GUARD) fail("read before the first guard", a);
        if (wa + 12 > (r < 3 ? (r + 1) * plane : bytes + WIN_GUARD)) fail("read enters the next plane", a);
        if (!err.empty()) break;
        if (wa + 12 - r * plane > max_end) max_end = wa + 12 - r * plane;
        for (int bx = 0; bx < 8; bx++)
          if (img[WIN_GUARD + b0 + bx] != Pf((long long)a + 4LL * by * ws + 4 * bx)) fail("corner byte is not P", a);
      }
    }
    printf("{\"width_step\": %d, \"data_size\": %d, \"lead\": %d, \"plane\": %d, \"pool_bytes\": %d, "
           "\"pitch\": %zu, \"interior\": %lld, \"max_read_end\": %d, \"ok\": %d, \"error\": \"%s\"}\n",
           ws, ds, lead, plane, bytes, l.pitch, interior, max_end, (int)err.empty(), err.c_str());
  }
  return 0;
}
