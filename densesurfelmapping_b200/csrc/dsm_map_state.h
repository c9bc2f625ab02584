// Private to the library: what the checkpoint file of dsm_io.cpp (dsm_map_save / dsm_map_load) needs to know about a
// context beyond the C ABI.  Defined in dsm_capi.cu; hidden, so neither is exported.
#pragma once
#include "../../include/dsm.h"

struct DsmMapInfo
{
    dsm_params params;       // as given to dsm_create
    dsm_constants constants; // the set in force (dsm_set_constants)
    int store_cap;           // the inactive store's reservation in surfels, 0 without one
    bool publish_in_flight;  // a dsm_publish_enqueue snapshot has not been waited for
};

__attribute__((visibility("hidden"))) int dsm_map_info(const dsm_ctx *ctx, DsmMapInfo *info);
// the host-side checks of dsm_inactive_load, in its order; touches nothing
__attribute__((visibility("hidden"))) int dsm_inactive_load_check(const dsm_ctx *ctx, const dsm_surfel_t *surfels, int n,
                                                                  const int32_t *kf_ofs_cnt, int n_segments);
