// keys.cuh — 256-bit sort keys (canonical Fr values, four little-endian u64 limbs) and the binary search over a column
// sorted by them: shared by the lookup argument (lookup.cu) and the lookup check (check.cu).
#pragma once
#include <cstdint>

namespace h2b {

struct Key256 {
    uint64_t l[4];
};
__device__ __forceinline__ int key_cmp(const Key256& a, const Key256& b) {
#pragma unroll
    for (int i = 3; i >= 0; i--) {
        if (a.l[i] < b.l[i]) return -1;
        if (a.l[i] > b.l[i]) return 1;
    }
    return 0;
}
__device__ __forceinline__ Key256 key_load(const uint64_t* p, size_t i) {
    const ulonglong2* q = reinterpret_cast<const ulonglong2*>(p + 4 * i);
    ulonglong2 a = q[0], b = q[1];
    return Key256{{a.x, a.y, b.x, b.y}};
}

// is `key` present in the sorted column `col` (n canonical keys)?
__device__ __forceinline__ bool sorted_contains(const uint64_t* col, uint32_t n, const Key256& key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (key_cmp(key_load(col, mid), key) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && key_cmp(key_load(col, lo), key) == 0;
}

}  // namespace h2b
