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

// The sections of one checkpoint file, in file order
struct DsmMapSections
{
    const dsm_surfel_t *pool;
    int n_pool;
    const dsm_surfel_t *store;
    int n_store;
    const int32_t *table; // [n_segments][3]: keyframe, offset, count
    int n_segments;
    const void *extra;
    size_t extra_bytes;
};
// The one writer of the file (dsm_io.cpp), for dsm_map_save and the checkpoint thread: header from `info`, the sections,
// the checksum; under a temporary name, flushed to the disk and renamed over `path`.  DSM_E_IO leaves nothing under path.
__attribute__((visibility("hidden"))) int dsm_map_write(const char *path, const DsmMapInfo &info, const DsmMapSections &s);
