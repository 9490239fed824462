// hector_node_plan (csrc/hector_node_plan.cuh) on the host, for tests/test_hector_node_plan.py.  One request per stdin
// line: B, then per node: started next_tick_ns period_ns n_scans and its n_scans stamps as sec nsec pairs.  One JSON line
// per request: the node's cuts, ticks and clock after the call, the part count and every part's [begin, end) per node.
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/hector_node_plan.cuh"

using namespace b2s;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    int B = 0;
    in >> B;
    std::vector<HectorNodeClock> clock((size_t)B);
    std::vector<int64_t> period((size_t)B);
    std::vector<int32_t> n((size_t)B);
    std::vector<uint32_t> stamps;
    for (int b = 0; b < B; b++) {
      int started = 0;
      long long next = 0, per = 0;
      in >> started >> next >> per >> n[(size_t)b];
      clock[(size_t)b].started = started != 0;
      clock[(size_t)b].next_tick_ns = next;
      period[(size_t)b] = per;
      for (int i = 0; i < 2 * n[(size_t)b]; i++) {
        unsigned long v = 0;
        in >> v;
        stamps.push_back((uint32_t)v);
      }
    }
    const HectorNodePlan p = hector_node_plan(B, n.data(), stamps.data(), clock.data(), period.data());
    std::printf("{\"n_parts\": %d, \"nodes\": [", p.n_parts);
    for (int b = 0; b < B; b++) {
      std::printf("%s{\"cuts\": [", b ? ", " : "");
      for (size_t k = 0; k < p.cuts[(size_t)b].size(); k++) std::printf("%s%d", k ? ", " : "", p.cuts[(size_t)b][k]);
      std::printf("], \"ticks\": [");
      for (size_t k = 0; k < p.ticks[(size_t)b].size(); k++)
        std::printf("%s%lld", k ? ", " : "", (long long)p.ticks[(size_t)b][k]);
      std::printf("], \"started\": %d, \"next_tick\": %lld, \"parts\": [", p.after[(size_t)b].started ? 1 : 0,
                  (long long)p.after[(size_t)b].next_tick_ns);
      for (int k = 0; k < p.n_parts; k++)
        std::printf("%s[%d, %d]", k ? ", " : "", p.begin[(size_t)k * B + b], p.end[(size_t)k * B + b]);
      std::printf("]}");
    }
    std::printf("]}\n");
  }
  return 0;
}
