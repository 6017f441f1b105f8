// The segment -> group map of the grouped kernels that cut every group into fixed-size segments counted from the
// group's own first row: K15's partitions of 32 rows and K6's chains of 1024 rows.  sbase [n_groups + 1] is the exclusive
// scan of the groups' segment counts, so group g owns segments [sbase[g], sbase[g + 1]).
#pragma once
#include <cstdint>

namespace pdsb {
namespace {

// sgrp[k] = the group of segment k: the last g with sbase[g] <= k (an empty group shares its sbase with the next)
__global__ void segment_groups(const int64_t* __restrict__ sbase, int64_t n_groups, int64_t nseg, int64_t* __restrict__ sgrp) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nseg; k += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n_groups;                 // sbase[lo] <= k < sbase[hi]
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (__ldg(sbase + mid) <= k) lo = mid; else hi = mid; }
    sgrp[k] = lo;
  }
}

}  // namespace
}  // namespace pdsb
