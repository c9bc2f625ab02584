// Private to the library: what the checkpoint file of dsm_io.cpp (dsm_map_save / dsm_map_load) needs to know about a
// context beyond the C ABI.  Defined in dsm_capi.cu; hidden, so neither is exported.
#pragma once
#include <vector>

#include "../../include/dsm.h"

struct DsmMapInfo
{
    dsm_params params;       // as given to dsm_create
    dsm_constants constants; // the set in force (dsm_set_constants)
    int store_cap;           // the inactive store's reservation in surfels, 0 without one
    bool publish_in_flight;  // a dsm_publish_enqueue snapshot has not been waited for
    bool field_in_flight;    // a dsm_field_enqueue field has not been waited for
    int view_rays;           // rays per view (dsm_num_seeds) after dsm_checkpoint_views_enable, else 0
};

__attribute__((visibility("hidden"))) int dsm_map_info(const dsm_ctx *ctx, DsmMapInfo *info);
// the host-side checks of dsm_inactive_load, in its order; touches nothing
__attribute__((visibility("hidden"))) int dsm_inactive_load_check(const dsm_ctx *ctx, const dsm_surfel_t *surfels, int n,
                                                                  const int32_t *kf_ofs_cnt, int n_segments);

// the host-side checks of a views section (DESIGN.md §8.18) in its load order, touching nothing: DSM_E_CAPACITY for a
// slot >= max_views, DSM_E_INVALID for a ray dsm_views_capture cannot have written
__attribute__((visibility("hidden"))) int dsm_views_load_check(const dsm_ctx *ctx, const int32_t *slots, int n, const void *rays);
// Replaces the captured views by slots[0 .. n) with their rays ([n][dsm_num_seeds] float4, packed); every other slot
// becomes unfilled.  Synchronises.
__attribute__((visibility("hidden"))) int dsm_views_load(dsm_ctx *ctx, const int32_t *slots, int n, const void *rays);
// The filled slots, ascending, and their rays packed in that order, read in stream order.  Synchronises.
__attribute__((visibility("hidden"))) int dsm_views_download(dsm_ctx *ctx, std::vector<int32_t> &slots, std::vector<uint8_t> &rays);

// The sections of one checkpoint file, in file order.  rays_per_view > 0 makes it a version-2 file with a views section
// of n_views slots (ascending) after the table, view_rays[i] pointing at the rays_per_view float4 of view_slots[i].
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
    const int32_t *view_slots;
    int n_views;
    const void *const *view_rays;
    int rays_per_view;
};
// The one writer of the file (dsm_io.cpp), for dsm_map_save and the checkpoint thread: header from `info`, the sections,
// the checksum; under a temporary name, flushed to the disk and renamed over `path`.  DSM_E_IO leaves nothing under path.
// *checksum / *bytes (optional): the file's trailing checksum and its length.
__attribute__((visibility("hidden"))) int dsm_map_write(const char *path, const DsmMapInfo &info, const DsmMapSections &s,
                                                        uint64_t *checksum = nullptr, uint64_t *bytes = nullptr);

// The journal beside a base file (dsm_checkpoint_enqueue_incremental, DESIGN.md §8.6).  dsm_journal_start replaces
// <path>.journal by a header that names the base's checksum (temporary name, fsync, rename); *bytes is its length.
// rays_per_view > 0: the journal of a version-2 base, whose records carry views.
__attribute__((visibility("hidden"))) int dsm_journal_start(const char *path, uint64_t base_checksum, int rays_per_view, uint64_t *bytes);
// One record: the chunks of 256 surfels that changed since the previous state, in ascending order, each section's chunk c
// read at 11264 * c bytes from its base (the last chunk of a section cut at its size), then the whole table and extra.
// In the journal of a version-2 base, the views captured since the previous state: view_rays[i] points at the
// rays_per_view float4 of view_slots[i] (ascending).
struct DsmJournalRecord
{
    uint64_t sequence, prev_checksum;
    int n_pool, n_store, n_segments;
    const int32_t *pool_chunks; // [k_pool]
    int k_pool;
    const int32_t *store_chunks; // [k_store]
    int k_store;
    const uint8_t *pool, *store;
    const int32_t *table;
    const void *extra;
    size_t extra_bytes;
    const int32_t *view_slots;
    int k_views;
    const void *const *view_rays;
    int rays_per_view;
};
// Appends the record to <path>.journal, which must be `journal_bytes` long, and flushes it to the disk.  DSM_E_IO leaves
// the journal at its old length as far as it can.  *checksum / *bytes: the record's own checksum and its length.
__attribute__((visibility("hidden"))) int dsm_journal_append(const char *path, uint64_t journal_bytes, const DsmJournalRecord &r,
                                                             uint64_t *checksum, uint64_t *bytes);
// dsm_map_load and dsm_inactive_load tell the checkpoint that the map was replaced: the next incremental one is a base
__attribute__((visibility("hidden"))) void dsm_checkpoint_map_replaced(dsm_ctx *ctx);
