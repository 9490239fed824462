// libstdc++'s std::sort (bits/stl_algo.h, bits/stl_heap.h), restated step for step for one thread, host or device.
//
// lesson1's feature picker (feature_detection.cc:149-150) sorts {value, index} pairs by value with std::sort and then
// takes the top of the range.  std::sort is not stable, so which of several equal values ends up on top is decided by
// the exact sequence of moves libstdc++ makes.  Reproducing the picks bit for bit under ties therefore means making
// that sequence of moves:
//   - __introsort_loop: while the range has more than 16 elements, partition it around the median of three (moved to
//     `first`) with the unguarded partition, recurse on the right part and loop on the left; the depth limit is
//     2 * floor(log2 n) and, when it runs out, the range is heap-sorted (__partial_sort with middle == last, i.e.
//     __make_heap then __sort_heap, both through __adjust_heap / __push_heap);
//   - __final_insertion_sort: a guarded insertion sort of the first 16 elements, then an unguarded one of the rest.
// The recursion becomes an explicit stack: the subranges are disjoint, so the order they are processed in does not
// change the result.  T needs a `value` member compared with `<`; every other member just moves with it.
// tests/introsort_check.cpp checks the permutation against the host's std::sort.
#pragma once

#if defined(__CUDACC__)
#define B2S_HD __host__ __device__ __forceinline__
#else
#define B2S_HD inline
#endif

namespace b2s {
namespace introsort_detail {

constexpr int THRESHOLD = 16;  // _S_threshold
constexpr int STACK = 64;      // pending ranges: at most one per level of the depth limit, 2 * 31 + 1 for an int length

template <class T>
B2S_HD bool less(const T &a, const T &b) { return a.value < b.value; }

template <class T>
B2S_HD void swap(T *a, T *b) {
  const T t = *a;
  *a = *b;
  *b = t;
}

B2S_HD int lg(int n) {  // std::__lg
  int k = 0;
  while (n >>= 1) k++;
  return k;
}

template <class T>
B2S_HD void move_median_to_first(T *result, T *a, T *b, T *c) {
  if (less(*a, *b)) {
    if (less(*b, *c)) swap(result, b);
    else if (less(*a, *c)) swap(result, c);
    else swap(result, a);
  } else if (less(*a, *c)) swap(result, a);
  else if (less(*b, *c)) swap(result, c);
  else swap(result, b);
}

template <class T>
B2S_HD T *unguarded_partition(T *first, T *last, const T *pivot) {
  for (;;) {
    while (less(*first, *pivot)) ++first;
    --last;
    while (less(*pivot, *last)) --last;
    if (!(first < last)) return first;
    swap(first, last);
    ++first;
  }
}

template <class T>
B2S_HD void push_heap(T *first, int hole, int top, T value) {
  int parent = (hole - 1) / 2;
  while (hole > top && less(first[parent], value)) {
    first[hole] = first[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  first[hole] = value;
}

template <class T>
B2S_HD void adjust_heap(T *first, int hole, int len, T value) {
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (less(first[child], first[child - 1])) child--;
    first[hole] = first[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    first[hole] = first[child - 1];
    hole = child - 1;
  }
  push_heap(first, hole, top, value);
}

template <class T>
B2S_HD void heap_sort(T *first, T *last) {  // __partial_sort(first, last, last): __make_heap, then __sort_heap
  const int len = (int)(last - first);
  if (len >= 2)
    for (int parent = (len - 2) / 2;; parent--) {
      adjust_heap(first, parent, len, first[parent]);
      if (parent == 0) break;
    }
  while (last - first > 1) {  // __sort_heap: __pop_heap(first, last - 1, last - 1)
    --last;
    const T value = *last;
    *last = *first;
    adjust_heap(first, 0, (int)(last - first), value);
  }
}

template <class T>
B2S_HD void unguarded_linear_insert(T *last) {
  const T val = *last;
  T *next = last - 1;
  while (less(val, *next)) {
    *last = *next;
    last = next;
    --next;
  }
  *last = val;
}

template <class T>
B2S_HD void insertion_sort(T *first, T *last) {
  if (first == last) return;
  for (T *i = first + 1; i != last; ++i) {
    if (less(*i, *first)) {
      const T val = *i;
      for (T *p = i; p != first; --p) *p = *(p - 1);  // move_backward(first, i, i + 1)
      *first = val;
    } else {
      unguarded_linear_insert(i);
    }
  }
}

}  // namespace introsort_detail

// std::sort(first, last, [](a, b) { return a.value < b.value; }).  Returns how many ranges fell back to the heap sort
// (0 on almost every input; a median-of-three killer sequence reaches it).
template <class T>
B2S_HD int introsort(T *first, T *last) {
  namespace d = introsort_detail;
  if (first == last) return 0;
  int heap_fallbacks = 0;
  // pending (first, last, depth limit) as offsets; depths strictly fall towards the top, so at most 2 * 31 + 1 entries
  int stack[d::STACK][3];
  int top = 0, lo = 0, hi = (int)(last - first), depth = 2 * d::lg(hi);
  for (;;) {  // __introsort_loop on [lo, hi); the recursion on each right part becomes a push
    while (hi - lo > d::THRESHOLD) {
      if (depth == 0) {
        d::heap_sort(first + lo, first + hi);
        heap_fallbacks++;
        break;
      }
      --depth;
      T *mid = first + lo + (hi - lo) / 2;  // __unguarded_partition_pivot
      d::move_median_to_first(first + lo, first + lo + 1, mid, first + hi - 1);
      const int cut = (int)(d::unguarded_partition(first + lo + 1, first + hi, first + lo) - first);
      stack[top][0] = cut;
      stack[top][1] = hi;
      stack[top][2] = depth;
      top++;
      hi = cut;
    }
    if (top == 0) break;
    --top;
    lo = stack[top][0];
    hi = stack[top][1];
    depth = stack[top][2];
  }
  if (last - first > d::THRESHOLD) {  // __final_insertion_sort
    d::insertion_sort(first, first + d::THRESHOLD);
    for (T *i = first + d::THRESHOLD; i != last; ++i) d::unguarded_linear_insert(i);
  } else {
    d::insertion_sort(first, last);
  }
  return heap_fallbacks;
}

}  // namespace b2s

#undef B2S_HD
