// ob_cub.cuh -- CUB device-wide sorts and scans of the C-ABI entry points, with their temporary storage taken from the
// call's Staging.  An op is one CUB call bound to its arguments, written as the CUB call without the temporary
// storage: sort_pairs(keys_in, keys_out, values_in, values_out, n, [decomposer,] begin_bit, end_bit, stream).  Each
// argument keeps its type, so a call compiles the same CUB kernels (NumItemsT included) as a direct call would.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "ob_api_common.h"

namespace ob {
namespace {

template <typename... A>
auto sort_pairs(A... a) {
    return [=](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortPairs(tmp, bytes, a...); };
}
template <typename... A>
auto sort_keys(A... a) {
    return [=](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortKeys(tmp, bytes, a...); };
}
template <typename... A>
auto inclusive_sum(A... a) {
    return [=](void* tmp, size_t& bytes) { return cub::DeviceScan::InclusiveSum(tmp, bytes, a...); };
}
template <typename... A>
auto exclusive_sum(A... a) {
    return [=](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, a...); };
}

// One block of temporary storage, sized for the largest of the ops given to the constructor, for ops that run one
// after another on one stream.  A failed size query, allocation or call is recorded in the Staging, and once it holds
// an error nothing is queried, allocated or run.
class CubTemp {
   public:
    template <typename... Op>
    explicit CubTemp(Staging& stg, const Op&... ops) : stg_(stg) {
        (size(ops), ...);
        tmp_ = stg_.scratch<void>(bytes_);
    }
    // run one op on the block: returns the Staging's error
    template <typename Op>
    cudaError_t run(const Op& op) {
        if (!stg_.error()) stg_.check(op(tmp_, bytes_));
        return stg_.error();
    }

   private:
    template <typename Op>
    void size(const Op& op) {
        size_t need = 0;
        if (!stg_.error() && stg_.check(op(nullptr, need)) == cudaSuccess) bytes_ = std::max(bytes_, need);
    }
    Staging& stg_;
    size_t bytes_ = 0;
    void* tmp_ = nullptr;
};

// one op with a block of its own
template <typename Op>
cudaError_t cub_run(Staging& stg, const Op& op) {
    return CubTemp(stg, op).run(op);
}

// radix bits that hold 0..v
int bits_for(unsigned long long v) {
    int b = 1;
    while (b < 64 && (v >> b) != 0) ++b;
    return b;
}

}  // namespace
}  // namespace ob
