// attn_sets.cuh -- the key set of a query and the query set of a key for the three attention kinds, shared by the SIMT attention
// kernels (forward, JVP and both VJP passes) and their launchers.  Plain C++ when __CUDACC__ is not defined, so a host program can
// enumerate the sets and check them against the reference's attention masks.
#pragma once

#include "kdiffusion_b200.h"

#ifndef __CUDACC__
#include <algorithm>
#define __host__
#define __device__
#endif

namespace kdb {

#ifndef __CUDACC__
using std::max;
using std::min;
#endif

// The keys of query token q, enumerated per attention type.
struct KeySet {
  int type, h, w, param, shift;
  int qi, qj;           // query coordinates
  int r0, c0;           // neighbourhood origin
  int wi, wj, lqi, lqj; // shifted-window: window index and local query coords (rolled frame)
  __host__ __device__ static int count(int type, int h, int w, int param) { return type == KDB_ATTN_GLOBAL ? h * w : param * param; }
  __host__ __device__ int count() const { return count(type, h, w, param); }
  __host__ __device__ void init(int type_, int h_, int w_, int param_, int shift_, int q) {
    type = type_; h = h_; w = w_; param = param_; shift = shift_;
    qi = q / w; qj = q - qi * w;
    if (type == KDB_ATTN_NEIGHBORHOOD) {
      r0 = min(max(qi - param / 2, 0), h - param);
      c0 = min(max(qj - param / 2, 0), w - param);
    } else if (type == KDB_ATTN_SHIFTED_WINDOW) {
      const int ri = (qi + shift) % h, rj = (qj + shift) % w;   // position in the rolled image (:274)
      wi = ri / param; wj = rj / param; lqi = ri - wi * param; lqj = rj - wj * param;
    }
  }
  // token index of key j, or -1 if masked out
  __host__ __device__ int token(int j) const {
    if (type == KDB_ATTN_GLOBAL) return j;
    const int a = j / param, b = j - a * param;
    if (type == KDB_ATTN_NEIGHBORHOOD) return (r0 + a) * w + (c0 + b);
    if (shift > 0) {   // seam mask (:300-315): only the first window row/col contains wrapped tokens
      if (wi == 0 && ((lqi < shift) != (a < shift))) return -1;
      if (wj == 0 && ((lqj < shift) != (b < shift))) return -1;
    }
    const int oi = (wi * param + a - shift + h) % h, oj = (wj * param + b - shift + w) % w;
    return oi * w + oj;
  }
};

// The inverse of KeySet: the queries whose key set contains key token `kt` (the key-centric pass of the attention VJP).
//   global: every query.
//   shifted window: the queries of the key's rolled window on the key's side of the seam (the seam mask is symmetric).
//   neighbourhood: per axis the queries with s(i) <= a < s(i) + k, s(i) = clamp(i - k/2, 0, n - k); s is monotone, so they form one
//   contiguous range.  On an axis of n >= 2k tokens it holds k queries inside the grid and up to 3 (k/2) + 1 near a border; on a
//   shorter axis the windows clamped at the two borders overlap, and a middle key can be seen by all n queries.
struct QuerySet {
  int type, h, w, param, shift;
  int i0, j0, ni, nj;   // neighbourhood: query row/column ranges [i0, i0+ni) x [j0, j0+nj)
  int wi, wj, la, lb;   // shifted-window: the key's window and local coords (rolled frame)
  // the most queries that see one key of a neighbourhood axis of n >= k tokens (reached by some key for odd k, an upper bound for even k)
  __host__ __device__ static int axis_max(int n, int k) { return n <= 2 * k - 1 ? n : 3 * (k / 2) + 1; }
  __host__ __device__ static int max_count(int type, int h, int w, int param) {
    if (type == KDB_ATTN_GLOBAL) return h * w;
    if (type == KDB_ATTN_NEIGHBORHOOD) return axis_max(h, param) * axis_max(w, param);
    return param * param;
  }
  __host__ __device__ static void range(int a, int n, int k, int& lo, int& cnt) {
    lo = n;
    int hi = -1;
    for (int i = max(0, a - 2 * k); i <= min(n - 1, a + 2 * k); ++i) {
      const int s = min(max(i - k / 2, 0), n - k);
      if (s <= a && a < s + k) {
        lo = min(lo, i);
        hi = max(hi, i);
      }
    }
    cnt = hi - lo + 1;
  }
  __host__ __device__ int count() const {
    if (type == KDB_ATTN_GLOBAL) return h * w;
    if (type == KDB_ATTN_NEIGHBORHOOD) return ni * nj;
    return param * param;
  }
  __host__ __device__ void init(int type_, int h_, int w_, int param_, int shift_, int kt) {
    type = type_; h = h_; w = w_; param = param_; shift = shift_;
    const int ki = kt / w, kj = kt - (kt / w) * w;
    if (type == KDB_ATTN_NEIGHBORHOOD) {
      range(ki, h, param, i0, ni);
      range(kj, w, param, j0, nj);
    } else if (type == KDB_ATTN_SHIFTED_WINDOW) {
      const int ri = (ki + shift) % h, rj = (kj + shift) % w;
      wi = ri / param; wj = rj / param; la = ri - wi * param; lb = rj - wj * param;
    }
  }
  // token index of query t, or -1 if the seam mask hides the key from it
  __host__ __device__ int token(int t) const {
    if (type == KDB_ATTN_GLOBAL) return t;
    if (type == KDB_ATTN_NEIGHBORHOOD) return (i0 + t / nj) * w + (j0 + t % nj);
    const int a = t / param, b = t - a * param;   // the query's local coords in the key's window
    if (shift > 0) {
      if (wi == 0 && ((a < shift) != (la < shift))) return -1;
      if (wj == 0 && ((b < shift) != (lb < shift))) return -1;
    }
    const int oi = (wi * param + a - shift + h) % h, oj = (wj * param + b - shift + w) % w;
    return oi * w + oj;
  }
};

}  // namespace kdb
