// scan.cuh — the u32 exclusive scan of the grid build (icp.cu, DESIGN.md §4.2), also used by the point-cloud
// extraction (extract.cu).  The scan kernels stay in icp.cu; this header carries its host entry point and tile size.
#pragma once

#include "reduce.cuh"   // kThreads

namespace o3db {

static constexpr int kScanItems = 8;
static constexpr int kScanTile = kThreads * kScanItems;

// Exclusive scan of u32 data[0..n) in place; data[n] receives the (32-bit) total.  data has n+1 entries; scratch
// has ceil(n/kScanTile) entries.  Three launches on `st`.
int exclusive_scan_u32(unsigned* data, int64_t n, unsigned* scratch, cudaStream_t st);

}  // namespace o3db
