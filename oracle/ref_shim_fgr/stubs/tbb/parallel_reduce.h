// ref_shim_fgr stub (test infrastructure): tbb::parallel_reduce on one thread.  The imperative form runs the one
// body over the whole range, which is what TBB does with a single worker: the range is cut into chunks, but with no
// thief the body is never split, so one body sees every chunk in order.
#pragma once
#include "tbb/blocked_range.h"
namespace tbb {
struct split {};
template <typename Range, typename Body>
void parallel_reduce(const Range& range, Body& body) {
    body(range);
}
template <typename Range, typename Value, typename Body, typename Join>
Value parallel_reduce(const Range& range, const Value& identity, const Body& body, const Join&) {
    return body(range, identity);
}
}  // namespace tbb
