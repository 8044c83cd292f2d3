// Work items of a probed-list scan, built on the device from a probe table [nq, nprobe] of list ids: the probe table is
// inverted into per-list query sets, and every (list, chunk of <= kIvfChunk queries probing it) becomes one item.
// Shared by the IVF scan (flat_ip.cu) and the AH code scan (ah.cu).  Nothing is read back to the host: the item count
// stays in device memory.
#pragma once

#include <stdint.h>

namespace mmb {
namespace {

constexpr int kIvfChunk = 128;      // probing queries per work item
constexpr int kIvfMaxProbe = 1024;

// probes per list
__global__ void ivf_count_kernel(const int64_t* __restrict__ probes, int64_t n_pairs, int64_t nlist, int* __restrict__ cnt) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_pairs; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = probes[p];
    if (l >= 0 && l < nlist) atomicAdd(cnt + l, 1);
  }
}

// One block of 1024 threads: exclusive scans of the probe counts (first gathered row of each list) and of the item
// counts ceil(cnt / kIvfChunk) (first item of each list); the total item count goes to *n_items.  Thread t scans a
// contiguous segment, so the result does not depend on scheduling.
__global__ void __launch_bounds__(1024) ivf_scan_kernel(const int* __restrict__ cnt, int64_t nlist,
                                                        int* __restrict__ row_base, int* __restrict__ item_base,
                                                        int* __restrict__ n_items) {
  __shared__ int s_rows[1024], s_items[1024];
  const int t = threadIdx.x;
  const int64_t seg = (nlist + 1023) / 1024, lo = min(nlist, t * seg), hi = min(nlist, lo + seg);
  int rows = 0, items = 0;
  for (int64_t l = lo; l < hi; ++l) { rows += cnt[l]; items += (cnt[l] + kIvfChunk - 1) / kIvfChunk; }
  s_rows[t] = rows;
  s_items[t] = items;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {   // inclusive Hillis-Steele scan
    const int r = t >= o ? s_rows[t - o] : 0, i = t >= o ? s_items[t - o] : 0;
    __syncthreads();
    s_rows[t] += r;
    s_items[t] += i;
    __syncthreads();
  }
  rows = s_rows[t] - rows;
  items = s_items[t] - items;
  for (int64_t l = lo; l < hi; ++l) {
    row_base[l] = rows;
    item_base[l] = items;
    rows += cnt[l];
    items += (cnt[l] + kIvfChunk - 1) / kIvfChunk;
  }
  if (t == 1023) *n_items = s_items[1023];
}

// The work items of every list: (list, first gathered row, rows), in list order.
__global__ void ivf_items_kernel(const int* __restrict__ cnt, int64_t nlist, const int* __restrict__ row_base,
                                 const int* __restrict__ item_base, int4* __restrict__ items) {
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < nlist; l += (int64_t)gridDim.x * blockDim.x) {
    const int c = cnt[l];
    for (int j = 0; j * kIvfChunk < c; ++j)
      items[item_base[l] + j] = make_int4((int)l, row_base[l] + j * kIvfChunk, min(kIvfChunk, c - j * kIvfChunk), 0);
  }
}

}  // namespace
}  // namespace mmb
