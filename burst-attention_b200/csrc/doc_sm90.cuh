// Packed documents (cu_seqlens) for the doc tile kernels (kDoc in fwd_sm90.cuh / bwd_sm90.cuh): the document of a
// full-sequence position, and the interval of a view's rows or keys that lies in one document.  A view's index i sits
// at position pos0 + pstride i, so the indices of one document form one interval of the view.
#pragma once
#include <stdint.h>

namespace ba {

// Positions are int32 (cu_seqlens is): the entry points check that every row's and key's position fits.

// the document of full-sequence position x (the last d with cu[d] <= x, so that cu[d] <= x < cu[d + 1] for x
// inside the sequence; zero-length documents are skipped), clamped to [0, n_docs - 1]
__device__ __forceinline__ int doc_of(const int* cu, int n_docs, int x) {
  int lo = 0, hi = n_docs;  // invariant: cu[lo] <= x (or lo = 0), and the answer is < hi
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cu + mid) <= x) lo = mid;
    else hi = mid;
  }
  return lo;
}

// ceil((x - pos0) / pstride) clamped to [0, n]: the first index of a view (position pos0 + pstride i) at or
// after position x
__device__ __forceinline__ int doc_view_index(int x, int pos0, int pstride, int n) {
  if (x <= pos0) return 0;
  const unsigned i = ((unsigned)(x - pos0) + (unsigned)(pstride - 1)) / (unsigned)pstride;
  return i >= (unsigned)n ? n : (int)i;
}

// the indices [*lo, *hi) of a view of n tokens from position pos0 (keys for a row, or rows for a key) that share a
// document with position x
__device__ __forceinline__ void doc_interval(int x, const int* cu, int n_docs, int pos0, int pstride, int n, int* lo,
                                             int* hi) {
  const int d = doc_of(cu, n_docs, x);
  *lo = doc_view_index(__ldg(cu + d), pos0, pstride, n);
  *hi = doc_view_index(__ldg(cu + d + 1), pos0, pstride, n);
}

}  // namespace ba
