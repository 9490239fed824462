/*
 * feature_oracle.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * CPU restatement of lesson1's corner picker, LaserScan::ScanCallback (reference/lesson1/src/feature_detection.cc:77-179),
 * for the contract of b2s_feature_detect (include/b200slam.h).  The sort is the host's std::sort, as in the node.
 * Built on its own by oracle/features_port.py (-O2, no FMA contraction, like the reference's catkin build).
 *
 * Beyond the node's output it reports, per scan, which sectors had a tied cut (the 20th pick equal in value to the
 * first value left out, so that the picks depend on std::sort's order among equal values) and how many sector sorts
 * fell back to heap sort, so that tests can show their cases reach those paths.  The second figure comes from the
 * restated introsort (csrc/introsort.cuh) run on a copy; its permutation is checked against std::sort's here as well.
 */
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <functional>
#include <vector>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/introsort.cuh"

namespace {

constexpr int MAX_SCAN_COUNT = 1500;  // max_scan_count (:23)

struct smoothness_t {  // :25-29
  float value;
  size_t index;
};

struct by_value {  // :32-38
  bool operator()(smoothness_t const &l, smoothness_t const &r) const { return l.value < r.value; }
};

}  // namespace

extern "C" {

/* One scan: ranges[n] (n <= 1500), edge_threshold (the node's 1.0, :69).  out_ranges[n] = corner_scan.ranges[0, n);
 * out_curvature[n] (may be NULL) = c_i at beam orig(i), NaN where the stencil computed nothing.
 * info[4] = {picks or -1 (NaN curvature), tied-cut sector mask (bit j = sector j), heap-sort fallbacks,
 *            1 if the restated introsort disagreed with std::sort on some sector}.
 * With info NULL the diagnostics are skipped (for timing the restatement itself) and the count is not returned.
 * Returns 0, or -1 for n outside [0, 1500]. */
int orc_feature_detect(int n, const float *ranges, float edge_threshold, float *out_ranges, float *out_curvature,
                       int32_t *info) {
  if (n < 0 || n > MAX_SCAN_COUNT) return -1;
  int32_t scratch[4];
  const bool diag = info != nullptr;
  if (!diag) info = scratch;
  info[0] = info[1] = info[2] = info[3] = 0;
  for (int i = 0; i < n; i++) out_ranges[i] = 0.0f;
  const uint32_t qnan_bits = 0x7fc00000u;  // the one NaN of the contract's curvature row
  float qnan;
  std::memcpy(&qnan, &qnan_bits, sizeof qnan);
  if (out_curvature)
    for (int i = 0; i < n; i++) out_curvature[i] = qnan;
  // :93-106 valid readings in beam order; orig[k] is map_index[k]
  std::vector<float> v;
  std::vector<int> orig;
  for (int i = 0; i < n; i++)
    if (std::isfinite(ranges[i])) {
      orig.push_back(i);
      v.push_back(ranges[i]);
    }
  const int count = (int)v.size();
  // :81 value-initialised {0, 0}; :112-124 the stencil, left to right in float
  std::vector<smoothness_t> S(std::max(count, 1), smoothness_t{0.0f, 0});
  bool nan = false;
  for (int i = 5; i < count - 5; i++) {
    float diff_range = v[i - 5] + v[i - 4] + v[i - 3] + v[i - 2] + v[i - 1] - v[i] * 10 + v[i + 1] + v[i + 2] + v[i + 3] +
                       v[i + 4] + v[i + 5];
    const float c = diff_range * diff_range;
    S[i].value = c;
    S[i].index = (size_t)i;
    if (out_curvature) out_curvature[orig[i]] = std::isnan(c) ? qnan : c;
    nan = nan || std::isnan(c);
  }
  if (nan) {  // std::sort's ordering breaks down on NaN; the contract reports the scan instead of guessing
    info[0] = -1;
    return 0;
  }
  int picks = 0;
  for (int j = 0; j < 6; j++) {  // :139-171
    const int s = (0 * (6 - j) + count * j) / 6;
    const int e = (0 * (5 - j) + count * (j + 1)) / 6 - 1;
    if (s >= e) continue;
    std::vector<smoothness_t> copy;
    if (diag) {
      // is the cut tied?  K picks come from the sorted range [s, e) after S[e] (considered first, unsorted)
      std::vector<float> q;
      for (int k = s; k < e; k++)
        if (S[k].value > edge_threshold) q.push_back(S[k].value);
      const int K = S[e].value > edge_threshold ? 19 : 20;
      if ((int)q.size() > K) {
        std::sort(q.begin(), q.end(), std::greater<float>());
        if (q[K - 1] == q[K]) info[1] |= 1 << j;
      }
      copy.assign(S.begin() + s, S.begin() + e);
      info[2] += b2s::introsort(copy.data(), copy.data() + copy.size());
    }
    // :149-150 the node's sort: half-open, S[e] is not sorted
    std::sort(S.begin() + s, S.begin() + e, by_value());
    if (diag)
      for (int k = s; k < e; k++)
        if (copy[k - s].index != S[k].index) info[3] = 1;
    // :152-170 the walk from S[e] down
    int largestPickedNum = 0;
    for (int k = e; k >= s; k--) {
      const int index = (int)S[k].index;
      if (S[k].value > edge_threshold) {
        largestPickedNum++;
        if (largestPickedNum <= 20) {
          out_ranges[orig[index]] = ranges[orig[index]];
          picks++;
        } else {
          break;
        }
      }
    }
  }
  info[0] = picks;
  return 0;
}

/* McIlroy's adversary ("A Killer Adversary for Quicksort", 1999) against this host's std::sort on n elements:
 * out[n] gets values whose order drives the median-of-three pivot to its worst case, so that an introsort of that
 * order exhausts its depth limit and falls back to heap sort.  Only the order of the values matters.  Elements with
 * top[i] != 0 (top may be NULL) are fixed beforehand as equal maxima, n + 1; the adversary orders the others. */
void orc_feature_killer_order(int n, const uint8_t *top, float *out) {
  std::vector<int> val(n, n), order(n);
  int solid = 0, candidate = 0;
  const int gas = n;
  for (int i = 0; i < n; i++)
    if (top && top[i]) val[i] = n + 1;
  for (int i = 0; i < n; i++) order[i] = i;
  std::sort(order.begin(), order.end(), [&](int x, int y) {
    if (val[x] == gas && val[y] == gas) val[x == candidate ? x : y] = solid++;
    if (val[x] == gas) candidate = x;
    else if (val[y] == gas) candidate = y;
    return val[x] < val[y];
  });
  for (int i = 0; i < n; i++) out[i] = (float)val[i];
}

}  // extern "C"
