// grl_param_list.cuh -- lists of differently sized images passed to a kernel by value, in its kernel parameters.
//
// The list kernels (image_list.cu, dataset_u8.cu, awgn.cu, jpeg.cu, resize.cu) take a host array of image descriptors.
// A launch carries up to N records of them by value in the 4 KB of kernel parameters, so a call needs no device copy
// and no host sync; a longer list takes several launches on the caller's stream.  A kernel finds its record from a grid
// index, or with record_of from a flat index over the whole launch.  Records are read inline from the parameters: a
// reference or pointer into them passed to a function the compiler does not inline makes every thread copy the whole
// list to local memory.
#pragma once

#include "grl_common.cuh"

namespace grl {

// Up to N records R of one launch; Other: the bytes of the launch's other kernel parameters.
template <class R, int N, int Other = 0>
struct ParamList {
  static constexpr int kCapacity = N;
  static_assert(sizeof(R) * N + Other <= 4096, "a launch's records and other parameters fit the kernel parameters");
  R at[N];
};

// Runs the n items of a list in launches of at most List::kCapacity records.  add(L.at[j], j, i) writes item i's record
// as record j of the launch and returns the work it brings, or -1 (only for j >= 1) when it would overflow the launch's
// flat indices, which starts the next launch with it.  launch(L, i0, m) runs items i0 .. i0 + m - 1; a launch whose
// items bring no work is skipped.  Returns the first error.
template <class List, class Add, class Launch>
int launch_list(int n, Add add, Launch launch) {
  List L = {};  // records past a launch's m are never read
  for (int i0 = 0, m; i0 < n; i0 += m) {
    long long work = 0;
    for (m = 0; i0 + m < n && m < List::kCapacity; ++m) {
      const long long w = add(L.at[m], m, i0 + m);
      if (w < 0) break;
      work += w;
    }
    if (work == 0) continue;
    const int rc = launch(L, i0, m);
    if (rc != GRL_OK) return rc;
  }
  return GRL_OK;
}

// The record that owns flat index t of a launch whose m records start at first[0] = 0 <= first[1] <= ...: the last
// j < m with first[j] <= t.
__device__ __forceinline__ int record_of(const int* first, int m, int t) {
  int lo = 0, hi = m - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The list arguments of a call: n >= 0 items and, unless the list is empty, non-null host arrays.
inline int check_list_args(int n, bool arrays, const char* items, const char* what) {
  GRL_REQUIRE(n >= 0 && (arrays || n == 0), "%s: null %s list (n = %d)", what, items, n);
  return GRL_OK;
}

// The (source, destination) pairs of a list made from 8-bit images: source i is a GRL_IMAGE_U8 of at least 1 x 1,
// destination i has dst_kind and the size dst_size(source i) = {H, W}, and both have data (an empty destination may
// not).  limit(source i, i) checks the call's own bounds.
template <class Size, class Limit>
int check_u8_pairs(const GrlImageRef* src, const GrlImageRef* dst, int n, int dst_kind, Size dst_size, Limit limit,
                   const char* what) {
  static const char* const kKinds[] = {"GRL_IMAGE_F32", "GRL_IMAGE_U8", "GRL_IMAGE_RGGB"};
  int rc = check_list_args(n, src && dst, "image", what);
  for (int i = 0; rc == GRL_OK && i < n; ++i) {
    const GrlImageRef &s = src[i], &d = dst[i];
    const int2 need = dst_size(s);
    GRL_REQUIRE(s.kind == GRL_IMAGE_U8 && d.kind == dst_kind, "%s: image %d: kinds %d / %d, need GRL_IMAGE_U8 -> %s", what,
                i, s.kind, d.kind, kKinds[dst_kind]);
    GRL_REQUIRE(s.H >= 1 && s.W >= 1 && d.H == need.x && d.W == need.y,
                "%s: image %d: sizes %d x %d -> %d x %d, need %d x %d", what, i, s.H, s.W, d.H, d.W, need.x, need.y);
    GRL_REQUIRE(s.data && (d.data || (long long)d.H * d.W == 0), "%s: image %d: null data", what, i);
    rc = limit(s, i);
  }
  return rc;
}

}  // namespace grl
