// prefix.cuh — the copies of a prefix state cache (include/rwkv_b200.h, "Prefix state cache"; the index is
// prefix_index.h). A cache's pool holds xy, aa, bb and dd of `capacity` entries, each array [capacity][L][E] f64 like
// the slot arrays. The passes write snapshots into it (PassDesc::snap, k_pf_wkv, k_pf_store_state); this kernel moves
// whole states between entries and slots.
#pragma once

#include "common.cuh"

namespace rk {

constexpr unsigned long long kPrefixZero = ~0ull; // a pair's entry: write the zero state
constexpr int kPrefixThreads = 256, kPrefixPerThread = 4; // 16-byte words per thread of a chunk

struct PrefixCopyArgs {
    double *pool[4];                 // xy, aa, bb, dd of entry 0
    double *slot[5];                 // xy, aa, bb, pp, dd of slot 0
    size_t LE;                       // doubles per array of one entry or slot (even: E is a multiple of 16)
    const unsigned long long *pairs; // [n][2] {entry or kPrefixZero, slot}
    int restore;                     // 1: entry -> slot, pp = 0 (5 arrays); 0: slot -> entry (4 arrays)
};

// grid (pairs, arrays, chunks): block (i, a, x) copies chunk x of array a of pair i in 16-byte words (the pair count is
// bounded by max_gpt only, so it takes the grid's x dimension). A restore writes
// all five arrays of the slot (pp and, for kPrefixZero, the others from zero), so the slot holds exactly the state a
// zeroed slot reaches after the entry's tokens: no forward writes pp.
__global__ void __launch_bounds__(kPrefixThreads) k_prefix_copy(const __grid_constant__ PrefixCopyArgs a) {
    static constexpr int kSlotArray[5] = {0, 1, 2, 4, 3}; // pool array (and pp last) -> slot array
    const int arr = blockIdx.y;
    const unsigned long long e = a.pairs[2 * blockIdx.x], s = a.pairs[2 * blockIdx.x + 1];
    double2 *sl = reinterpret_cast<double2 *>(a.slot[kSlotArray[arr]] + (size_t)s * a.LE);
    const double2 *en = arr < 4 && e != kPrefixZero ? reinterpret_cast<const double2 *>(a.pool[arr] + (size_t)e * a.LE) : nullptr;
    const size_t n2 = a.LE / 2;
    const size_t j0 = (size_t)blockIdx.z * kPrefixThreads * kPrefixPerThread + threadIdx.x;
#pragma unroll
    for (int k = 0; k < kPrefixPerThread; ++k) {
        const size_t j = j0 + (size_t)k * kPrefixThreads;
        if (j >= n2) break;
        if (a.restore) sl[j] = en ? en[j] : make_double2(0.0, 0.0);
        else reinterpret_cast<double2 *>(a.pool[arr] + (size_t)e * a.LE)[j] = sl[j];
    }
}

inline dim3 prefix_copy_grid(size_t LE, bool restore, unsigned long long n) {
    const size_t per_block = (size_t)kPrefixThreads * kPrefixPerThread;
    return dim3((unsigned)n, restore ? 5u : 4u, (unsigned)((LE / 2 + per_block - 1) / per_block)); // z <= 100 at 14B
}

} // namespace rk
