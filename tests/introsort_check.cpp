// csrc/introsort.cuh against the host's std::sort: for every length 0 .. max_len and several input families, the two
// must leave the {value, index} pairs in the same order (the same index permutation, ties included).  Prints one JSON
// line: cases run, mismatches, and how many cases reached the heap-sort fallback.
//
//   g++ -O2 -std=c++17 introsort_check.cpp -o introsort_check && ./introsort_check 300
#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/introsort.cuh"

namespace {

struct Item {  // smoothness_t (feature_detection.cc:25-29)
  float value;
  size_t index;
};

// McIlroy's adversary ("A Killer Adversary for Quicksort", 1999) run against std::sort: values are frozen as late as
// the comparisons allow, which drives the median-of-three pivot to the worst case and the introsort into its heap sort
std::vector<float> killer(int n) {
  std::vector<int> val(n, n), order(n);
  int solid = 0, candidate = 0;
  const int gas = n;
  for (int i = 0; i < n; i++) order[i] = i;
  std::sort(order.begin(), order.end(), [&](int x, int y) {
    if (val[x] == gas && val[y] == gas) val[x == candidate ? x : y] = solid++;
    if (val[x] == gas) candidate = x;
    else if (val[y] == gas) candidate = y;
    return val[x] < val[y];
  });
  return std::vector<float>(val.begin(), val.end());
}

std::vector<float> family(int f, int n, std::mt19937 &rng) {
  std::vector<float> v(n);
  switch (f) {
    case 0: for (auto &x : v) x = std::uniform_real_distribution<float>(0.0f, 1.0f)(rng); break;  // random
    case 1: for (auto &x : v) x = 1.0f; break;                                                     // all equal
    case 2: for (auto &x : v) x = (float)std::uniform_int_distribution<int>(0, 2)(rng); break;     // three values
    case 3: for (auto &x : v) x = (float)std::uniform_int_distribution<int>(0, 7)(rng); break;     // eight values
    case 4: for (int i = 0; i < n; i++) v[i] = (float)i; break;                                    // sorted
    case 5: for (int i = 0; i < n; i++) v[i] = (float)(n - i); break;                              // reversed
    case 6: for (int i = 0; i < n; i++) v[i] = (float)std::min(i, n - 1 - i); break;               // organ pipe
    case 7: v = killer(n); break;                                                                  // adversary
    default: for (int i = 0; i < n; i++) v[i] = (float)(i % 5); break;                             // sawtooth
  }
  return v;
}

}  // namespace

int main(int argc, char **argv) {
  const int max_len = argc > 1 ? std::atoi(argv[1]) : 300;
  const int families = 9, reps = 4;
  long cases = 0, mismatches = 0, fallback_cases = 0, killer_fallbacks = 0;
  int first_bad_len = -1, first_bad_family = -1;
  std::mt19937 rng(12345);
  for (int n = 0; n <= max_len; n++)
    for (int f = 0; f < families; f++)
      for (int rep = 0; rep < (f == 0 || f == 2 || f == 3 ? reps : 1); rep++) {
        const std::vector<float> v = family(f, n, rng);
        std::vector<Item> a(n), b(n);
        for (int i = 0; i < n; i++) a[i] = b[i] = Item{v[i], (size_t)i};
        std::sort(a.begin(), a.end(), [](const Item &l, const Item &r) { return l.value < r.value; });
        const int fb = b2s::introsort(b.data(), b.data() + n);
        cases++;
        bool same = true;
        for (int i = 0; i < n; i++) same = same && a[i].index == b[i].index && a[i].value == b[i].value;
        if (!same) {
          mismatches++;
          if (first_bad_len < 0) { first_bad_len = n; first_bad_family = f; }
        }
        if (fb) {
          fallback_cases++;
          if (f == 7) killer_fallbacks++;
        }
      }
  std::printf("{\"cases\": %ld, \"mismatches\": %ld, \"fallback_cases\": %ld, \"killer_fallbacks\": %ld, "
              "\"first_bad_len\": %d, \"first_bad_family\": %d}\n",
              cases, mismatches, fallback_cases, killer_fallbacks, first_bad_len, first_bad_family);
  return 0;
}
