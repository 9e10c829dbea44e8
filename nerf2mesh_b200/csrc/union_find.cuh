// union_find.cuh -- the lock-free union-find shared by the mesh clean-up (meshclean.cu) and the UV atlas (atlas.cu): parent[x] <= x,
// so the root of a class is its lowest element whatever the order the unions run in.
#pragma once

#include <stdint.h>

namespace n2m {

__device__ __forceinline__ int32_t uf_find(int32_t* parent, int32_t x) {
    volatile int32_t* p = parent;
    while (true) {
        const int32_t y = p[x];
        if (y == x) return x;
        const int32_t z = p[y];
        if (z != y) p[x] = z;                  // path halving: z is still an ancestor of x
        x = y;
    }
}
// once every union is done: the root, without writes (a path-halving write racing a label store could leave a non-root behind)
__device__ __forceinline__ int32_t uf_root(const int32_t* parent, int32_t x) {
    int32_t y;
    while ((y = parent[x]) != x) x = y;
    return x;
}
__device__ __forceinline__ void uf_union(int32_t* parent, int32_t a, int32_t b) {
    while (true) {
        a = uf_find(parent, a); b = uf_find(parent, b);
        if (a == b) return;
        if (a < b) { const int32_t t = a; a = b; b = t; }
        if (atomicCAS(parent + a, a, b) == a) return;
    }
}

}  // namespace n2m
