// The union kernel of every whole-frame labelling (locate.cu, edges.cu, ct.cu); see ccl.cuh.
#include "ccl.cuh"

namespace epid {

__global__ void k_ccl_union(int H, int W, int conn8, int* __restrict__ parent) {
    const int f = blockIdx.y, HW = H * W;
    int* par = parent + (size_t)f * HW;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        if (par[i] < 0) continue;
        const int y = i / W, x = i - y * W;
        ccl_join(par, i, x, y, W, conn8 != 0);
    }
}

}  // namespace epid
