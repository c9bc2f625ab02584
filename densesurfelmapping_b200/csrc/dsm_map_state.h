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
    bool field_in_flight;    // a dsm_field_enqueue field has not been waited for
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
// *checksum / *bytes (optional): the file's trailing checksum and its length.
__attribute__((visibility("hidden"))) int dsm_map_write(const char *path, const DsmMapInfo &info, const DsmMapSections &s,
                                                        uint64_t *checksum = nullptr, uint64_t *bytes = nullptr);

// The journal beside a base file (dsm_checkpoint_enqueue_incremental, DESIGN.md §8.6).  dsm_journal_start replaces
// <path>.journal by a header that names the base's checksum (temporary name, fsync, rename); *bytes is its length.
__attribute__((visibility("hidden"))) int dsm_journal_start(const char *path, uint64_t base_checksum, uint64_t *bytes);
// One record: the chunks of 256 surfels that changed since the previous state, in ascending order, each section's chunk c
// read at 11264 * c bytes from its base (the last chunk of a section cut at its size), then the whole table and extra.
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
};
// Appends the record to <path>.journal, which must be `journal_bytes` long, and flushes it to the disk.  DSM_E_IO leaves
// the journal at its old length as far as it can.  *checksum / *bytes: the record's own checksum and its length.
__attribute__((visibility("hidden"))) int dsm_journal_append(const char *path, uint64_t journal_bytes, const DsmJournalRecord &r,
                                                             uint64_t *checksum, uint64_t *bytes);
// dsm_map_load and dsm_inactive_load tell the checkpoint that the map was replaced: the next incremental one is a base
__attribute__((visibility("hidden"))) void dsm_checkpoint_map_replaced(dsm_ctx *ctx);
