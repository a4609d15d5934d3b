// tn_sort.cuh -- what every CUB sort, scan and select of the library shares, and the search the kernels that read sorted keys share.
#pragma once
#include "tn_common.cuh"

namespace tn {

// Runs one CUB device algorithm on the temporary storage `tmp`: call(nullptr, bytes) sizes it, tmp grows to that, call(tmp.p, bytes)
// runs.  `call` states the algorithm's arguments once, so the size query and the run always describe the same call.
template <class F>
int cub_run(DevArray<uint8_t> &tmp, F &&call) {
    size_t bytes = 0;
    TN_CUDA(call(nullptr, bytes));
    TN_TRY(tmp.grow(bytes));
    TN_CUDA(call(tmp.p, bytes));
    return TN_OK;
}

// end_bit of a radix sort whose keys are at most max_key: the bit width of max_key, at least 1
inline int radix_end_bit(uint64_t max_key) { return 64 - __builtin_clzll(max_key | 1ull); }

// the first position in the ascending keys a[0, n) whose key is >= x (n if none)
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t *__restrict__ a, uint32_t n, uint32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid; }
    return lo;
}

}  // namespace tn
