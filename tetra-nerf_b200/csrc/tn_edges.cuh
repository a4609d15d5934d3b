// tn_edges.cuh -- the edges of a tetrahedron, as the refinement pass (tn_refine.cu) and the vertex adjacency (tn_smoothness.cu) see them.
#pragma once
#include <stdint.h>

namespace tn {

// the six edges of a tetrahedron as local vertex pairs
#define TN_TET_EDGES const int EA[6] = {0, 0, 0, 1, 1, 2}, EB[6] = {1, 2, 3, 2, 3, 3}

// the undirected edge {a, b} as one key: (min << 32) | max
__device__ __forceinline__ unsigned long long edge_key(uint32_t a, uint32_t b) {
    return a < b ? ((unsigned long long)a << 32) | b : ((unsigned long long)b << 32) | a;
}

}  // namespace tn
