// Windowed disk locator of wl.cu (internal interface): the k_wl_bb search of SizedDiskLocator over a list of items, each with its
// own source frame, pixel map and search parameters.
#pragma once
#include "common.cuh"

namespace epid {

// pixels of an item's source are read as I = (v - mn) / D (v: uint16 of the source frame); status != EPID_WL_OK skips the item
struct WlItemMap {
    int status;
    uint32_t mn, D;
};

size_t disk_items_scratch_bytes(int n_items);

// n items, one CTA each, results to d_res[i] (epid_disk_result, image coordinates).  `scratch`: disk_items_scratch_bytes(n) bytes of
// device memory; max_window_px: the largest search window edge of the items (sizes the shared-memory forest).
int launch_disk_items(epid_ctx* ctx, cudaStream_t st, void* scratch, int n, int H, int W, double dpmm, double max_window_px,
                      const uint16_t* const* d_src, const WlItemMap* d_maps, const epid_disk_params* d_loc, epid_disk_result* d_res);

}  // namespace epid
