// Union-find on a per-pixel parent array for 4-connected component labelling (postproc.cu, targets.cu).
// L[p] is p's parent (or a negative value for a pixel outside every component); a root is its own parent.
// uf_union always hangs the larger root under the smaller one, so the root of a component is its smallest linear
// index, i.e. its first pixel in raster order (what scipy.ndimage.label numbers by).
#pragma once

namespace hvn {

__device__ __forceinline__ int uf_find(const int *L, int a) {
    int r = a;
    while (true) {
        int p = L[r];
        if (p == r) return r;
        r = p;
    }
}
__device__ __forceinline__ void uf_union(int *L, int a, int b) {
    while (true) {
        a = uf_find(L, a);
        b = uf_find(L, b);
        if (a == b) return;
        if (a > b) { int t = a; a = b; b = t; }
        int old = atomicMin(&L[b], a);  // hang the larger root under the smaller one
        if (old == b) return;
        b = old;
    }
}

}  // namespace hvn
