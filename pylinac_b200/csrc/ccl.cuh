// Connected-component labelling by union-find on a parent array, shared by every labelling stage: roots are the smallest index of a
// component (= skimage / scipy label order), hooking by atomicMin, path halving.  A frame's parents are frame-local indices in
// [0, H * W), -1 off the foreground.
#pragma once

namespace epid {

__device__ __forceinline__ int gl_find(int* parent, int i) {
    while (true) {
        const int p = parent[i];
        if (p == i) return i;
        const int gp = parent[p];
        if (gp != p) atomicMin(&parent[i], gp);      // path halving; parents only ever decrease, so a concurrent hook is never lost
        i = p;
    }
}

__device__ __forceinline__ void gl_union(int* parent, int a, int b) {
    while (true) {
        a = gl_find(parent, a);
        b = gl_find(parent, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }      // hook the larger root under the smaller one
        const int old = atomicMin(&parent[a], b);
        if (old == a) return;
        a = old;
    }
}

// The one neighbour rule: joins foreground pixel i (column x, row y of a frame W wide) with its foreground neighbours earlier in
// raster order, the left and the upper one, and with conn8 the upper-left only when left and up are both background and the
// upper-right only when up is background.  The skipped diagonals change no component: with up set, the upper-left pixel is up's
// left neighbour and the upper-right one has up as its left neighbour; with left set, the upper-left pixel is left's upper neighbour.
__device__ __forceinline__ void ccl_join(int* par, int i, int x, int y, int W, bool conn8) {
    const bool l = x > 0 && par[i - 1] >= 0, u = y > 0 && par[i - W] >= 0;
    if (l) gl_union(par, i, i - 1);
    if (u) gl_union(par, i, i - W);
    if (conn8 && y > 0 && !u) {
        if (!l && x > 0 && par[i - W - 1] >= 0) gl_union(par, i, i - W - 1);
        if (x + 1 < W && par[i - W + 1] >= 0) gl_union(par, i, i - W + 1);
    }
}

// the root of foreground pixel i once every union of its frame has finished: roots no longer change, so the plain walk suffices
// (concurrent writes of a pixel's root into par only shorten it)
__device__ __forceinline__ int ccl_root(const int* par, int i) {
    int r = i;
    while (par[r] != r) r = par[r];
    return r;
}

// ccl_join over every foreground pixel of a batch of H x W frames (frame blockIdx.y, parents at parent + f * H * W), any grid.x and
// block size
__global__ void k_ccl_union(int H, int W, int conn8, int* __restrict__ parent);

}  // namespace epid
