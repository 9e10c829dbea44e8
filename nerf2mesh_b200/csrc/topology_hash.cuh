// topology_hash.cuh -- the edge hash of a triangle mesh (built by k_aa_topology, csrc/antialias.cu): open addressing over `slots`
// (a power of two), key (min, max) vertex of one undirected edge as a 64-bit word, kEmptyKey in a free slot, linear probing from
// topo_hash(key) & (slots - 1).  Shared by the antialias kernels and the stage-1 mesh regularisers (csrc/stage1.cu).
#pragma once

#include <stdint.h>

namespace n2m {

constexpr unsigned long long kEmptyKey = ~0ull;

__device__ __forceinline__ uint32_t aa_hash(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (uint32_t)k;
}

__device__ __forceinline__ unsigned long long edge_key(int a, int b) {
    return ((unsigned long long)(uint32_t)min(a, b) << 32) | (unsigned long long)(uint32_t)max(a, b);
}

// the slot of edge (a, b), or -1 when it is not in the hash
__device__ __forceinline__ int64_t topo_find(const unsigned long long* __restrict__ keys, uint32_t mask, int a, int b) {
    const unsigned long long key = edge_key(a, b);
    uint32_t h = aa_hash(key) & mask;
    for (uint32_t probe = 0; probe <= mask; ++probe) {
        const unsigned long long k = keys[h];
        if (k == key) return h;
        if (k == kEmptyKey) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}

}  // namespace n2m
