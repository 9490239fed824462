// The publish schedule of lesson4's Hector SLAM node handle (hector_node.cu) over one call, for every node of the handle,
// and the launch parts it splits the call into.  Host only, no CUDA runtime: tests/hector_node_plan_check.cu runs it on
// the CPU against the restatement's schedule.
//
// The schedule (include/b200slam.h, DESIGN.md §7): tick 0 is the stamp of the node's first scan ever handed in; before
// a scan whose stamp >= the next tick the map is published once, stamped with that tick, and the next tick becomes the
// first tick strictly after the scan's stamp.  The period is Duration::fromSec(map_pub_period) (ros_math.cuh) in ns.
//
// The parts: part 0 holds every node's scans before its first publish; part k >= 1 holds node b's scans from its k-th
// publish up to its next (or the end of its call), and is empty for a node with fewer than k publishes.  So there are
// 1 + (the largest publish count) parts, each node's scans fall into them in order, and a node publishing before part k
// has all of its earlier scans in parts 0 ... k - 1.
#pragma once

#include <stdint.h>

#include <algorithm>
#include <vector>

namespace b2s {

// one node's schedule, carried from call to call
struct HectorNodeClock {
  bool started = false;      // tick 0 set (a scan was handed in)
  int64_t next_tick_ns = 0;  // the next tick, once started
};

struct HectorNodePlan {
  int batch = 0, n_parts = 1;
  std::vector<std::vector<int>> cuts;       // [B]: the scans of the node's call a publish precedes, ascending
  std::vector<std::vector<int64_t>> ticks;  // [B]: their ticks (ns)
  std::vector<HectorNodeClock> after;       // [B]: each node's schedule once the call is done
  std::vector<int> begin, end;              // [n_parts][B]: node b's scans [begin, end) of its call in part k
};

inline int64_t hector_stamp_ns(const uint32_t *s) { return (int64_t)s[0] * 1000000000LL + (int64_t)s[1]; }

// n_scans [B]; stamps [sum n_scans][2] (sec, nsec), node-major; clock [B] before the call; period_ns [B] > 0
inline HectorNodePlan hector_node_plan(int batch, const int32_t *n_scans, const uint32_t *stamps,
                                       const HectorNodeClock *clock, const int64_t *period_ns) {
  HectorNodePlan p;
  p.batch = batch;
  p.cuts.resize((size_t)batch);
  p.ticks.resize((size_t)batch);
  p.after.assign(clock, clock + batch);
  size_t first = 0;
  int most = 0;
  for (int b = 0; b < batch; b++) {
    HectorNodeClock &c = p.after[(size_t)b];
    for (int i = 0; i < n_scans[b]; i++) {
      const int64_t s = hector_stamp_ns(stamps + 2 * (first + (size_t)i));
      if (!c.started) {
        c.started = true;
        c.next_tick_ns = s;  // tick 0
      }
      if (s >= c.next_tick_ns) {
        p.cuts[(size_t)b].push_back(i);
        p.ticks[(size_t)b].push_back(c.next_tick_ns);
        c.next_tick_ns += ((s - c.next_tick_ns) / period_ns[b] + 1) * period_ns[b];  // the first tick strictly after s
      }
    }
    first += (size_t)n_scans[b];
    most = std::max(most, (int)p.cuts[(size_t)b].size());
  }
  p.n_parts = 1 + most;
  p.begin.assign((size_t)p.n_parts * batch, 0);
  p.end.assign((size_t)p.n_parts * batch, 0);
  for (int b = 0; b < batch; b++) {
    const std::vector<int> &c = p.cuts[(size_t)b];
    for (int k = 0; k < p.n_parts; k++) {
      // part k runs from the k-th publish (scan 0 for k = 0) to the next; past the node's last publish it is empty
      const int lo = k == 0 ? 0 : (k <= (int)c.size() ? c[(size_t)k - 1] : n_scans[b]);
      const int hi = k < (int)c.size() ? c[(size_t)k] : n_scans[b];
      p.begin[(size_t)k * batch + b] = lo;
      p.end[(size_t)k * batch + b] = hi;
    }
  }
  return p;
}

}  // namespace b2s
