// Private to the library: the context behind the opaque `dsm_ctx` of include/dsm.h, shared by the translation units
// that hold its entry points (dsm_capi.cu: the map, the field and checkpoints; dsm_comm.cu: multi-GPU gather over NCCL;
// dsm_field.cu, dsm_frontier.cu, dsm_reach.cu, dsm_gain.cu, dsm_viewpoint.cu, dsm_tour.cu, dsm_trajectory.cu,
// dsm_heading.cu and dsm_terrain.cu: the planner jobs, each beside its kernels), and the lifecycle those jobs share.
#pragma once
#include "dsm_device.cuh"
#include "dsm_map_state.h"
#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

struct DsmComm; // multi-GPU state (dsm_comm.cu), nullptr until dsm_comm_init

// Owning handles: each releases its resource exactly once, when it is reset or destroyed.  Internal to the library:
// hidden, so that their template instantiations stay out of its exported symbols.
#pragma GCC visibility push(hidden)
template <typename H, cudaError_t (*release)(H)>
struct Release
{
    void operator()(H h) const { release(h); }
};
template <typename T>
using DevPtr = std::unique_ptr<T, Release<void *, cudaFree>>;
using HostPtr = std::unique_ptr<void, Release<void *, cudaFreeHost>>;
using StreamPtr = std::unique_ptr<CUstream_st, Release<cudaStream_t, cudaStreamDestroy>>;
using EventPtr = std::unique_ptr<CUevent_st, Release<cudaEvent_t, cudaEventDestroy>>;
using GraphExecPtr = std::unique_ptr<CUgraphExec_st, Release<cudaGraphExec_t, cudaGraphExecDestroy>>;

// Every allocation, stream and event a context or communicator makes once and keeps for its lifetime.  The raw pointers
// and handles the code works with (and the DsmDev the kernels receive) are views; the owner releases them when its
// holder is deleted.  The holder's streams must be drained before that.
//
// The owner keeps its first failed call until take(): every call after it is a no-op that returns that failure, so a
// list of calls needs one check at its end.  An owner that outlives a failure takes it before its next call.
struct CudaOwner
{
    std::vector<DevPtr<void>> dev;
    std::vector<HostPtr> pinned;
    std::vector<StreamPtr> streams;
    std::vector<EventPtr> events;
    cudaError_t failed = cudaSuccess;

    // the first failure since the last take() (cudaSuccess: none), cleared
    cudaError_t take()
    {
        const cudaError_t e = failed;
        failed = cudaSuccess;
        return e;
    }
    template <typename T>
    cudaError_t device(T **p, size_t n, bool zero = false)
    {
        if (failed != cudaSuccess) return failed;
        cudaError_t e = cudaMalloc((void **)p, n * sizeof(T));
        if (e == cudaSuccess) dev.emplace_back(*p);
        if (e == cudaSuccess && zero) e = cudaMemset(*p, 0, n * sizeof(T));
        return failed = e;
    }
    template <typename T>
    cudaError_t host(T **p, size_t n)
    {
        if (failed != cudaSuccess) return failed;
        cudaError_t e = cudaMallocHost((void **)p, n * sizeof(T));
        if (e == cudaSuccess) pinned.emplace_back(*p);
        return failed = e;
    }
    // pinned host memory the device writes directly: *dev is its device alias
    template <typename T, typename D>
    cudaError_t mapped(T **p, D **dev, size_t n)
    {
        if (failed != cudaSuccess) return failed;
        cudaError_t e = cudaHostAlloc((void **)p, n * sizeof(T), cudaHostAllocMapped);
        if (e != cudaSuccess) return failed = e;
        pinned.emplace_back(*p);
        return failed = cudaHostGetDevicePointer((void **)dev, *p, 0);
    }
    cudaError_t stream(cudaStream_t *s, int priority = 0)
    {
        if (failed != cudaSuccess) return failed;
        cudaError_t e = cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority);
        if (e == cudaSuccess) streams.emplace_back(*s);
        return failed = e;
    }
    cudaError_t event(cudaEvent_t *ev, unsigned flags = cudaEventDisableTiming)
    {
        if (failed != cudaSuccess) return failed;
        cudaError_t e = cudaEventCreateWithFlags(ev, flags);
        if (e == cudaSuccess) events.emplace_back(*ev);
        return failed = e;
    }
};
#pragma GCC visibility pop
// The context types below hold these handles but keep default visibility (their own template instantiations stay
// exported as they are); GCC's warning about that mix does not matter for types that never cross the library boundary.
#pragma GCC diagnostic ignored "-Wattributes"

struct ProfRec
{
    int id;
    cudaEvent_t e0, e1;
};

// A captured kernel schedule, replayable while every launch parameter is unchanged.
struct GraphEntry
{
    int f0, nf, maxper, phase;
    const void *pool, *poolofs, *gate;
    GraphExecPtr exec;
};

// The inactive store (dsm_inactive_*): the attached_surfels of every pose outside the drift-free window, dense on the
// device in retirement order, with what the window step needs next to it.  dsm_inactive_reserve replaces it whole.  The
// (keyframe, offset, count) segment table and the store size live on the device (seg, win_hdr), and only the window step
// changes them; segs / size mirror them, exactly unless win_pending, and only res_sync refreshes the mirror.
struct InactStore
{
    CudaOwner own;                  // the device buffers below
    dsm_surfel_t *surfels = nullptr; // [cap]
    int4 *seg = nullptr;            // [cap] (keyframe, offset, count, scratch): a stored segment holds >= 1 surfel
    int32_t *blk = nullptr;         // [DSM_WINDOW_MAX_KEYS][blk_stride] per-key block counts over the pool
    int32_t *sync = nullptr;        // [dsm_win_sync_len(cap)] compaction flags
    int32_t *range = nullptr;       // [2] {first, last} of the range an export works on, set in stream order by k_set2
    // dsm_publish_*, allocated with the store once publishing is enabled: the inactive cloud as the host last received
    // it (device shadow, 16 B per reserved surfel) and its pinned host mirror with the device alias the kernel writes
    float4 *shadow = nullptr, *mirror_dev = nullptr; // [cap]
    dsm_point_t *mirror = nullptr;                   // [cap], host
    int cap = 0, blk_stride = 0;
    int size = 0;
    int upper = 0; // host-side upper bound of the store size (exact after a sync)
    struct Seg
    {
        int kf, ofs, cnt;
    };
    std::vector<Seg> segs;
};

// dsm_checkpoint_* (DESIGN.md §8.5): the device image k_map_snapshot writes in stream order, its pinned host twin
// k_map_drain fills on a low-priority stream, and the thread that writes the file.  The thread touches only the host
// image and the job below; the caller's thread owns everything else.
struct DsmCheckpoint
{
    CudaOwner own;                 // the drain stream and its events
    std::unique_ptr<CudaOwner> img; // the two images; dsm_inactive_reserve rebuilds them at the store's new size
    DsmSnapLayout lay{};
    uint8_t *dev = nullptr, *host = nullptr, *host_dev = nullptr; // device image, host image and its device alias
    cudaStream_t s_drain = nullptr;
    cudaEvent_t ev_snap = nullptr, ev_drain = nullptr; // after k_map_snapshot on the context's stream, after k_map_drain
    int drain_ctas = DSM_DRAIN_CTAS;
    int pool_chunks = 0, store_chunks = 0; // k_map_delta's flags after the image: one per 256-surfel chunk of each capacity
    bool pending = false; // enqueued and not yet retired by dsm_checkpoint_wait (caller's thread only)
    // dsm_checkpoint_enqueue_incremental (DESIGN.md §8.6), caller's thread: the device image has been written by something
    // other than the incremental chain since its last checkpoint (a full checkpoint, new images), or the map was replaced
    // or its constants changed; the next incremental checkpoint is a base
    bool stale = true;
    // the job, guarded by m: queued from dsm_checkpoint_enqueue until the thread has stored its result
    std::mutex m;
    std::condition_variable cv;
    bool queued = false, quit = false;
    int result = DSM_OK, err_frame = 0;
    enum Kind
    {
        FULL,   // dsm_checkpoint_enqueue: the version-1 file
        BASE,   // an incremental checkpoint that writes the file and a fresh journal header
        RECORD, // an incremental checkpoint that appends one record to the journal
    } kind = FULL;
    std::string path;
    std::vector<uint8_t> extra;
    DsmMapInfo info{};
    // the incremental chain as the thread left it: the base under chain_path ("" when the last incremental checkpoint
    // failed), the checksum of its last record (of the base without one), the next sequence number, and the two lengths
    std::string chain_path;
    uint64_t chain_sum = 0, sequence = 1, base_bytes = 0, journal_bytes = 0;
    std::vector<int32_t> chunks; // the thread's list of changed chunks
    // dsm_checkpoint_views_enable (DESIGN.md §8.18): the views section of the image, device and pinned [max_views][S],
    // allocated once both enables have run.  Caller's thread: vgen[s] the capture generation (DsmViews::gen) the
    // section holds for slot s, 0 for none; snap_slots the slots the last snapshot copied.  The job: view_slots, the
    // slots its file or record lists, read from vhost by slot.
    std::unique_ptr<CudaOwner> vimg;
    float4 *vdev = nullptr, *vhost = nullptr;
    std::vector<uint64_t> vgen;
    std::vector<int32_t> snap_slots, view_slots;
    std::thread worker; // last: started once the members above exist

    ~DsmCheckpoint()
    { // a queued write finishes (its file lands) before the thread ends
        {
            std::lock_guard<std::mutex> lk(m);
            quit = true;
        }
        cv.notify_all();
        if (worker.joinable()) worker.join();
    }
};

// dsm_field_signed_enable (DESIGN.md §8.16): the signed grid with its header words (dsm_device.cuh) and its pinned copy
struct DsmSignedField
{
    CudaOwner own;
    int32_t *grid = nullptr; // device
    float *host = nullptr;   // pinned [voxels]
};

// dsm_field_* (DESIGN.md §8.7): the occupancy grid, the distance grid with its header words, the pinned host copy of
// both and the event after the copy, all allocated by dsm_field_enable
struct DsmField
{
    CudaOwner own;
    DsmFieldGrid g{}; // voxel and size; origin and bounds of the latest request
    size_t voxels = 0, bytes = 0; // voxels of the grid; bytes of the distance grid with its header
    uint8_t *occ = nullptr;
    int32_t *dist = nullptr, *host = nullptr; // device grid, pinned copy
    cudaEvent_t ev = nullptr;
    bool in_flight = false; // enqueued and not yet waited for
    bool requested = false; // a field has been enqueued: the device grid is one a query may read
    bool resident = false;  // the latest request copies only its header words (dsm_field_enqueue_resident)
    bool known = false;     // the latest request is a known one (dsm_field_enqueue_known): its query view is DSM_FIELD_VIEW
    bool known_waited = false; // the last waited request is a known one, and no request has been enqueued since
    uint64_t requests = 0;     // field requests enqueued so far (dsm_reach_enqueue pairs a frontier job with its field)
    std::unique_ptr<DsmSignedField> sgn; // nullptr until dsm_field_signed_enable: every request from then on builds it
    bool signed_latest = false;          // the latest request built the signed grid
    bool signed_waited = false;          // the last waited request built it, and no request has been enqueued since
};

// dsm_views_* (DESIGN.md §8.9), allocated by dsm_views_enable: the captured rays of max_views slots, which slots hold a
// capture, the pinned host copy of a known request's state grid, and the pinned and device staging of its pose list
struct DsmViews
{
    CudaOwner own;
    int max_views = 0;
    float max_range = 0.f;
    float4 *rays = nullptr;       // device [max_views][S]: camera-space ray ends, w = 1, or w = 0 for a seed without one
    std::vector<uint8_t> filled;  // [max_views], caller's thread: the slot has been captured
    bool checkpointed = false;    // dsm_checkpoint_views_enable: every checkpoint carries the filled slots
    std::vector<uint64_t> gen;    // [max_views], caller's thread: a fresh number at every capture or load of the slot
    uint64_t gens = 0;            // the last number handed out
    uint8_t *state = nullptr;     // pinned [voxels]
    uint8_t *stage_host = nullptr, *stage_dev = nullptr; // double poses[max_views][12] | int32 slots[max_views]
    static size_t stage_bytes(int n) { return 12 * sizeof(double) * (size_t)n + sizeof(int32_t) * (size_t)n; }
};

// What every planner job (dsm_field_query_* and the jobs on the known field, DESIGN.md §8.8-8.15) holds besides its
// own buffers: their owner, the pinned copy of its packed result, and the event after that copy
struct DsmJob
{
    CudaOwner own;
    uint8_t *res_host = nullptr;
    cudaEvent_t ev = nullptr;
    bool in_flight = false; // enqueued and not yet waited for
    uint64_t request = 0;   // the DsmField::requests of the field the latest job read (0: no job yet, or a tour)
    const int32_t *words() const { return reinterpret_cast<const int32_t *>(res_host); } // the result's header
};

// dsm_field_query_* (DESIGN.md §8.8): the packed request (pinned staging and its device twin) and the device result at
// the capacities of dsm_field_query_enable; both layouts live in dsm_field.cu
struct DsmFieldQuery : DsmJob
{
    int max_points = 0, max_traj = 0, max_wp = 0;
    uint8_t *req_host = nullptr, *req_dev = nullptr, *res_dev = nullptr;
    int n_points = 0, n_traj = 0; // of the query in flight or last waited for
};

struct DsmFrontierAcc; // what k_frontier_reduce accumulates per table entry (dsm_frontier.cu)

// dsm_frontier_* (DESIGN.md §8.10), allocated by dsm_frontier_enable for the field's grid: the job's device buffers and
// its packed result, which the gain, viewpoint and reach jobs read as well
struct DsmFrontier : DsmJob
{
    int voxels = 0, max_comp = 0, max_clusters = 0, max_voxels = 0;
    int32_t *label = nullptr;                                   // [voxels]
    int32_t *roots = nullptr, *count = nullptr, *cmap = nullptr, *cid = nullptr; // [max_comp]
    int32_t *slot_comp = nullptr, *sizes = nullptr, *offs = nullptr; // [max_clusters]
    DsmFrontierAcc *acc = nullptr;                              // [max_clusters]
    int32_t *idx = nullptr;                                     // [max_voxels]
    uint32_t *keys = nullptr, *keys_alt = nullptr;              // [max_voxels]
    int32_t *blk = nullptr, *blk_ofs = nullptr;                 // one per CTA of the compactions
    uint8_t *res = nullptr;                                     // the packed result (dsm_device.cuh)
    void *temp = nullptr;                                       // CUB scratch
    size_t temp_bytes = 0;
    // byte offsets of the result's cluster table and member list
    static size_t table_at() { return 4 * (size_t)DSM_FRONTIER_WORDS; }
    size_t list_at() const { return table_at() + sizeof(dsm_frontier_cluster_t) * (size_t)max_clusters; }
};

// dsm_reach_* (DESIGN.md §8.11), allocated by dsm_reach_enable for the field's grid: the job's device buffers, the packed
// result (dsm_reach.cu), the goal staging and the cost grid's pinned copy.  A terrain job (§8.21) runs in the same
// buffers: its plane has no more cells than the field has voxels, nor more 32 x 16 tiles than the field has 8^3 ones.
struct DsmReach : DsmJob
{
    int voxels = 0, tiles = 0, tn[3] = {0, 0, 0}; // tn: tiles per axis
    int max_targets = 0, max_path = 0, max_rounds = 0, ctas = 0; // ctas: the persistent CTAs of a round
    int ctas_flat = 0;                            // those of a terrain job's round (dsm_reach_enqueue_terrain)
    uint8_t *trav = nullptr;                      // [voxels]
    uint32_t *cost[2] = {nullptr, nullptr};       // [voxels] each
    int32_t *stamp = nullptr;                     // [tiles]: the latest round a tile was scheduled for
    int32_t *sched[2] = {nullptr, nullptr};       // [tiles] each: round r's schedule is sched[r % 2]
    int32_t *count = nullptr;                     // [3]: round r's schedule length is count[r % 3]
    int32_t *goals = nullptr;                     // device [max_targets][3] goal voxels, staged from goals_host
    unsigned long long *best = nullptr;           // [max_targets] (cost << 32 | viewpoint)
    int32_t *member = nullptr;                    // [max_targets] the cluster member attaining best
    long long *len = nullptr, *ofs = nullptr;     // [max_targets] path lengths and their exclusive prefix sums
    uint8_t *res = nullptr;                       // the packed result
    void *temp = nullptr;                         // CUB scratch of the path-length scan
    size_t temp_bytes = 0;
    int32_t *goals_host = nullptr; // pinned [max_targets][3]
    uint32_t *cost_host = nullptr; // pinned [voxels]
    bool host_copy = false;
    uint64_t terrain = 0; // the DsmTerrain::enqueues of the terrain job the latest job ran on (0: a field job, or none)
};

// dsm_reach_matrix_* (DESIGN.md §8.13), allocated by dsm_reach_matrix_enable for the field's grid: the job's device
// buffers, the packed result (dsm_reach.cu) and the site staging.  Per (site, slot) the costs are a tile's 512 voxels in
// tile-local order (x fastest), at ((size_t)site * max_tiles + slot) * 512 of each buffer.  A terrain job (§8.22) runs
// in the same buffers: a 32 x 16 tile has 512 cells too, and its plane has no more of them than the field has 8^3 tiles.
struct DsmReachMatrix : DsmJob
{
    int voxels = 0, tiles = 0, tn[3] = {0, 0, 0};
    int max_sites = 0, max_tiles = 0, max_rounds = 0, ctas = 0; // ctas: the persistent CTAs of a round
    int ctas_flat = 0;                            // those of a terrain job's round (dsm_reach_matrix_enqueue_terrain)
    int32_t *flag = nullptr, *scan = nullptr;     // [tiles]: the tile is active, and the exclusive sum of the flags
    int32_t *slot = nullptr;                      // [tiles]: the tile's slot, -1 when inactive
    uint32_t *mask = nullptr;                     // [tiles][16]: the tile's traversable voxels, bit t of word t / 32
    int32_t *tile_of = nullptr;                   // [max_tiles]: the tile of a slot
    uint32_t *cost[2] = {nullptr, nullptr};       // [max_sites][max_tiles][512] each
    int32_t *stamp = nullptr;                     // [max_sites][max_tiles]: the latest round a slot was scheduled for
    int32_t *sched[2] = {nullptr, nullptr};       // [max_sites][max_tiles] each: round r's schedule is sched[r % 2]
    int32_t *count = nullptr;                     // [max_sites][3]: site i's round-r schedule length is count[3 i + r % 3]
    int32_t *rounds = nullptr, *reached = nullptr; // [max_sites]: the rounds with a non-empty schedule, the reached voxels
    int32_t *sites = nullptr;                     // device [max_sites][3] the points' voxels, staged from sites_host
    uint8_t *res = nullptr;                       // the packed result, room for max_sites
    void *temp = nullptr;                         // CUB scratch of the tile scan, for the field's and every flat count
    size_t temp_bytes = 0;
    int32_t *sites_host = nullptr; // pinned [max_sites][3]
    int n_sites = 0; // of the job in flight or last waited for
};

// dsm_gain_* (DESIGN.md §8.12), allocated by dsm_gain_enable for the field's grid: the pinned and device staging of
// max_views views, the cluster-slot grid and the device result (dsm_gain.cu)
struct DsmGain : DsmJob
{
    int max_views = 0;
    DsmGainView *views_host = nullptr, *views_dev = nullptr; // [max_views]
    int32_t *slot = nullptr;                                  // device [voxels]
    uint8_t *res = nullptr;
};

struct DsmVpCluster; // what k_vp_clusters leaves per requested cluster (dsm_viewpoint.cu)

// dsm_viewpoint_* (DESIGN.md §8.15), allocated by dsm_viewpoint_enable: the job's device buffers, the pinned staging of
// the request and its device twin, and the packed result (both layouts in dsm_viewpoint.cu)
struct DsmViewpoint : DsmJob
{
    int max_clusters = 0, max_candidates = 0, ctas = 0; // ctas: the persistent CTAs of k_vp_score
    int ctas_terrain = 0;                               // those of a terrain job's k_vp_score (dsm_viewpoint_enqueue_terrain)
    uint8_t *stage_host = nullptr, *stage_dev = nullptr;
    DsmVpCluster *cl = nullptr;               // [max_clusters]
    unsigned long long *key = nullptr;        // [max_candidates]: the candidate's ranking key, ~0 when it is no viewpoint
    int32_t *list = nullptr;                  // [max_candidates]: the reached candidates, cluster * n_offsets + offset
    int32_t *count = nullptr;                 // [1]: their number
    uint8_t *res = nullptr;                   // the packed result, room for max_clusters at top_k 16
    int n_clusters = 0, top_k = 0; // of the job in flight or last waited for
};

// dsm_tour_* (DESIGN.md §8.14), allocated by dsm_tour_enable: the pinned and device matrix of max_sites^2 entries, the
// starts' tours and the device result (dsm_tour.cu)
struct DsmTour : DsmJob
{
    int max_sites = 0, max_starts = 0;
    uint32_t *matrix_host = nullptr, *matrix = nullptr; // [max_sites^2] each
    int32_t *tours = nullptr;                           // device [max_starts][max_sites]
    uint8_t *res = nullptr;
    int n = 0, n_starts = 0; // of the job in flight or last waited for
};

// dsm_trajectory_* (DESIGN.md §8.17), allocated by dsm_trajectory_enable: the pinned and device staging of the request,
// the L-BFGS history (6 max_memory doubles per point) and the device result (both layouts in dsm_trajectory.cu)
struct DsmTrajectory : DsmJob
{
    int max_traj = 0, max_points = 0, max_memory = 0;
    uint8_t *stage_host = nullptr, *stage_dev = nullptr;
    double *hist = nullptr;
    uint8_t *res = nullptr;
    int n = 0, n_points = 0; // of the job in flight or last waited for
};

// dsm_heading_* (DESIGN.md §8.19), allocated by dsm_heading_enable: the pinned and device staging of the request, the
// successor table (64 int8 per sample) and the device result (both layouts in dsm_heading.cu)
struct DsmHeading : DsmJob
{
    int max_traj = 0, max_samples = 0;
    uint8_t *stage_host = nullptr, *stage_dev = nullptr;
    int8_t *succ = nullptr;
    uint8_t *res = nullptr;
    int n = 0, n_samples = 0, n_rot = 0; // of the job in flight or last waited for
};

// dsm_terrain_* (DESIGN.md §8.20), allocated by dsm_terrain_enable for the field's grid collapsed along the up axis: the
// device result (its layout in dsm_terrain.cu)
struct DsmTerrain : DsmJob
{
    int up = 0, cells = 0;
    int m[3] = {0, 0, 0};
    uint8_t *res = nullptr;
    int origin[3] = {0, 0, 0}, headroom = 0, max_step = 0; // of the job in flight or last waited for
    uint64_t enqueues = 0; // jobs enqueued so far: tells two terrain jobs on one field request apart (DsmReach::terrain)
    // byte offsets of the result's sections for C cells, which the terrain reach job reads as well:
    //   float clearance[C] | pad to dsm_field_header(C) words | int32 header[8] (a field header's words, dsm_device.cuh) |
    //   int16 level[C] | uint8 status[C] | uint8 step[C]
    static constexpr int HEADER_WORDS = 8;
    static size_t header_at(int cells) { return 4 * dsm_field_header((size_t)cells); }
    static size_t level_at(int cells) { return header_at(cells) + 4 * HEADER_WORDS; }
    static size_t status_at(int cells) { return level_at(cells) + 2 * (size_t)cells; }
    static size_t step_at(int cells) { return status_at(cells) + (size_t)cells; }
    static size_t res_bytes(int cells) { return step_at(cells) + (size_t)cells; }
};

// The plane of a terrain job as the jobs on it see it (DESIGN.md §8.21-8.23): n the plane (P, Q, 1), o the terrain job's
// origin; nf the field grid's extents and h0 < h1 its two in-plane axes, which map a field voxel to the cell of its column
struct ReachTerrainGrid : DsmFieldGrid
{
    int nf[3], h0, h1;
};

// The plane of terrain job tr on field grid fg: the plane (P, Q, 1) of fg's two axes h0 < h1 other than the up axis, at
// tr's origin
static inline ReachTerrainGrid reach_terrain_grid(const DsmFieldGrid &fg, const DsmTerrain &tr)
{
    const int a = std::abs(tr.up) - 1;
    ReachTerrainGrid g;
    static_cast<DsmFieldGrid &>(g) = fg;
    g.h0 = a == 0 ? 1 : 0, g.h1 = a == 2 ? 1 : 2;
    for (int k = 0; k < 3; k++) g.o[k] = tr.origin[k], g.nf[k] = fg.n[k];
    g.n[0] = fg.n[g.h0], g.n[1] = fg.n[g.h1], g.n[2] = 1;
    return g;
}

#define DSM_MAX_CHUNKS 4

struct dsm_ctx
{
    CudaOwner own; // the buffers, streams and events below (the caller's stream excepted)
    dsm_params p{};
    int device = 0;
    cudaStream_t stream = nullptr; // the caller's stream, or one of own.streams
    DsmComm *comm = nullptr;
    DsmDev d{};                    // geometry, constants and the batch-mode views of the buffers
    DsmMaps maps{};                // TMA descriptors of labels / depth / gray for the tile kernels
    int nb = 0;                    // frames in the current batch
    int n_pool = 0;                // local surfels in the current batch
    bool uploaded = false, ran = false;
    bool in_flight = false; // a dsm_fuse_batch_async batch has been enqueued and not yet waited for
    int stop_after = 0;     // debug: number of kernels to enqueue (<= 0: all)
    std::vector<GraphEntry> graphs; // CUDA-graph cache of the kernel schedule (launch-bound single-frame / small-chunk runs)
    bool use_graphs = true;
    // non-const views of what DsmDev holds, and buffers the kernels take as arguments
    uint8_t *gray = nullptr;
    float *depth = nullptr;
    dsm_surfel_t *pool_snap = nullptr; // second pool-sized buffer: batch snapshot, ordered output of the resident-pool exports
    int32_t *poolofs = nullptr, *refidx = nullptr;
    float *pose = nullptr, *ipose = nullptr;
    dsm_seed_t *seed_export = nullptr;
    float *kx = nullptr, *ky = nullptr;
    // packed staging of every call that takes images (stage_images; k_repack lays it out in gray / depth), copy streams
    uint8_t *gray_packed = nullptr; // [B][H][W]
    float *depth_packed = nullptr;  // [B][H][W]
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr, s_comp[DSM_MAX_CHUNKS] = {};
    cudaStream_t s_hi = nullptr; // highest priority: the frame-by-frame (latency-bound) phase of dsm_fuse_stream_resident
    cudaEvent_t ev_p2 = nullptr; // end of that phase, joined into the main stream
    // resident pool (stream mode)
    int res_upper = 0;   // host-side upper bound of the resident pool size (exact after a sync)
    bool res_active = false;
    int res_frame = 0;   // resident stream runs so far (alternates the staging halves)
    int32_t *res_ofs = nullptr; // device [4]: {0, resident pool size, error tag of dsm_fuse_stream_window, rejected frame}
    int *blkcnt = nullptr, *blkofs = nullptr, *nsel = nullptr; // ordered selection: per-block counts / offsets, total
    int32_t *holes = nullptr, *rc_src = nullptr, *rc_sync = nullptr; // fuse_map post-step (dsm_launch_pool_recycle)
    float *wmat = nullptr; // device copy of the 4x4 of dsm_pool_transform
    std::unique_ptr<InactStore> inact; // nullptr until dsm_inactive_reserve
    // dsm_fuse_stream_window: staged window lists (pinned h_win -> d_win, one table of win_len ints per staging half) and
    // the store's device header {size, segments, per-frame scratch x2}
    int32_t *h_win = nullptr, *d_win = nullptr, *win_hdr = nullptr;
    size_t win_len = 0;
    int win_tag = 0;          // tag of the latest windowed call (what a rejected frame writes into the error word)
    bool win_pending = false; // a window step since the last synchronisation: mirrors stale, error word unread
    cudaEvent_t ev_h2d[DSM_MAX_CHUNKS] = {}, ev_done[DSM_MAX_CHUNKS] = {}, ev_start = nullptr; // dsm_fuse_batch_async's chunks
    // the resident stream's staging halves: half_h2d[h] ends a run's input copy into half h; half_free[h] lies on the main
    // stream after every earlier use of half h (stream_run records it, see there)
    cudaEvent_t half_h2d[2] = {}, half_free[2] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[DSM_MAX_CHUNKS] = {}; // run_parts: fork / join of the parts on s_comp
    // frame slots [img_slot0, img_slot0 + img_n) hold the images of the most recent call that took images (img_n == 0: none
    // yet; hold_frames writes these with nb, uploaded and ran); dsm_frame_raw_cloud reads them, into raw_out (W*H points, allocated at its first call).  img_fit: that call's
    // schedule has run through the plane fit, so the slots' label codes and plane normals are complete;
    // dsm_frame_superpixel_image reads them, into spimg_out ([H][3*Wp] bytes, allocated at its first call)
    int img_slot0 = 0, img_n = 0;
    bool img_fit = false;
    float4 *raw_out = nullptr;
    uint8_t *spimg_out = nullptr;
    // dsm_publish_*: pinned, mapped active cloud [max_local_surfels] and snapshot header [DSM_PUB_WORDS] with their device
    // aliases, k_cloud_mirror's device state, the event that ends a snapshot.  The inactive side lives with the store.
    bool pub_on = false, pub_in_flight = false;
    dsm_point_t *pub_active = nullptr;
    float4 *pub_active_dev = nullptr;
    int32_t *pub_hdr = nullptr, *pub_hdr_dev = nullptr, *pub_state = nullptr;
    cudaEvent_t pub_ev = nullptr;
    std::unique_ptr<DsmCheckpoint> ckpt; // nullptr until dsm_checkpoint_enable
    std::unique_ptr<DsmField> field;     // nullptr until dsm_field_enable
    std::unique_ptr<DsmFieldQuery> field_query; // nullptr until dsm_field_query_enable
    std::unique_ptr<DsmViews> views;             // nullptr until dsm_views_enable
    std::unique_ptr<DsmFrontier> frontier;       // nullptr until dsm_frontier_enable
    std::unique_ptr<DsmReach> reach;             // nullptr until dsm_reach_enable
    std::unique_ptr<DsmReachMatrix> reach_matrix; // nullptr until dsm_reach_matrix_enable
    std::unique_ptr<DsmGain> gain;               // nullptr until dsm_gain_enable
    std::unique_ptr<DsmTour> tour;               // nullptr until dsm_tour_enable
    std::unique_ptr<DsmViewpoint> viewpoint;     // nullptr until dsm_viewpoint_enable
    std::unique_ptr<DsmTrajectory> trajectory;   // nullptr until dsm_trajectory_enable
    std::unique_ptr<DsmHeading> heading;         // nullptr until dsm_heading_enable
    std::unique_ptr<DsmTerrain> terrain;         // nullptr until dsm_terrain_enable
    int run_split = 2;          // sub-batches per dsm_batch_run (dsm_set_concurrency)
    // pinned host staging for the small per-batch tables
    float *h_pose = nullptr; // [2B][32]: pose then inverse; first half: the batch calls, second half: the resident stream
    int32_t *h_ofs = nullptr;
    int32_t *h_ref = nullptr; // [2B], halves as h_pose
    int32_t *h_sync = nullptr; // [8]: res_sync's readback of res_ofs and win_hdr
    // profiling
    uint32_t prof_mask = 0;
    std::vector<ProfRec> prof_pending;
    std::vector<cudaEvent_t> ev_free;
    float prof_ms[DSM_NUM_KERNELS] = {};
    int32_t prof_n[DSM_NUM_KERNELS] = {};
    char err[512] = {};
};

#define CK(call)                                                                                         \
    do                                                                                                   \
    {                                                                                                    \
        cudaError_t _e = (call);                                                                         \
        if (_e != cudaSuccess)                                                                           \
        {                                                                                                \
            snprintf(ctx->err, sizeof(ctx->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return DSM_E_CUDA;                                                                           \
        }                                                                                                \
    } while (0)

// ---- the lifecycle every snapshot, field and planner job shares ----
// The end of an enable: the new state is kept when every call of its owner succeeded and `ok`, else nothing is kept and
// a later call may try again
template <typename T>
static inline int keep(std::unique_ptr<T> &slot, std::unique_ptr<T> &fresh, bool ok = true)
{
    if (fresh->own.take() != cudaSuccess || !ok)
    {
        cudaGetLastError();
        return DSM_E_NOMEM; // nothing is kept: a later call may try again
    }
    slot = std::move(fresh);
    return DSM_OK;
}

// The latest field request if it is a known one (what every job on the known field reads), else nullptr
static inline const DsmField *known_field(const dsm_ctx *ctx)
{
    const DsmField *f = ctx->field.get();
    return f && f->requested && f->known ? f : nullptr;
}

// The pairing rule: the latest job of a kind (frontier, reach) read the latest field request
static inline bool read_latest(const DsmJob *j, const DsmField *f) { return j && j->request == f->requests; }

// The tail of an enqueue: one D2H copy of the used result bytes, the job's event, and the job in flight with the field
// request it read (0 for none)
static inline int submit(dsm_ctx *ctx, DsmJob &j, const void *res, size_t bytes, uint64_t request)
{
    CK(cudaMemcpyAsync(j.res_host, res, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaEventRecord(j.ev, ctx->stream));
    j.in_flight = true;
    j.request = request;
    return DSM_OK;
}

// The head of a wait (a job's or the field's): DSM_E_STATE without a request in flight, else its event waited for and
// the request retired
template <typename T>
static inline int wait_head(dsm_ctx *ctx, T *j)
{
    if (!j || !j->in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventSynchronize(j->ev));
    j->in_flight = false;
    return DSM_OK;
}

// The result of a wait whose header h holds the sticky error word of dsm_fuse_stream_window at h[tag] and the frame it
// rejected after it: DSM_OK without an error, else DSM_E_CAPACITY with the message that `call`'s `what` holds the frames
// before that one
static inline int capacity(dsm_ctx *ctx, const int32_t *h, int tag, const char *call, const char *what)
{
    if (h[tag] == 0) return DSM_OK;
    snprintf(ctx->err, sizeof(ctx->err), "%s: frame %d of a dsm_fuse_stream_window call did not fit the pool or the store; %s holds "
             "the frames before it", call, h[tag + 1], what);
    return DSM_E_CAPACITY;
}

// An info struct copied out of a result header, its reserved words zeroed
template <typename Info>
static inline void copy_info(Info *info, const int32_t *h)
{
    if (!info) return;
    std::memcpy(info, h, sizeof(Info));
    for (int32_t &w : info->reserved) w = 0;
}

// ---- host checks and staging shared by the jobs on a camera (gain, viewpoints, headings) or on splines (trajectories,
// headings) ----
// gain's camera checks (include/dsm.h): intrinsics, image size, the blocking rule and a range of at most 128 voxels
static inline bool gain_camera_ok(const dsm_gain_camera_t &c, double v)
{
    const double R = (double)c.max_range;
    return std::isfinite(c.fx) && c.fx > 0.0 && std::isfinite(c.fy) && c.fy > 0.0 && std::isfinite(c.cx) && std::isfinite(c.cy) &&
           c.width >= 1 && c.width <= 65536 && c.height >= 1 && c.height <= 65536 && (c.unknown_blocks == 0 || c.unknown_blocks == 1) &&
           std::isfinite(R) && R > 0.0 && R <= DSM_GAIN_MAX_RANGE_VOXELS * v;
}

// The grid voxels of view P's box: the bounding box of the image pyramid cut at depth max_range (the apex t and the
// four image corners (0 | width, 0 | height) at depth max_range) met with the cube around the range sphere, one voxel
// of padding, clipped to the grid.  Every centre that passes the frustum test lies in the truncated pyramid and in the
// sphere, so the box sizes the work and cannot change a count.  The pyramid holds them only for a rotation: a pose whose
// 3x3 part is not orthonormal within 1e-6 per entry of R^T R - I, or a corner that does not come out finite, leaves
// the cube alone (within that tolerance the pyramid moves by far less than the padding).
static inline void gain_box(const double *P, const dsm_gain_camera_t &c, const DsmFieldGrid &g, DsmGainView &V)
{
    const double R = (double)c.max_range, v = (double)g.voxel;
    double plo[3], phi[3];
    bool finite = true;
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++)
            finite = finite && std::fabs(((P[a] * P[b] + P[4 + a] * P[4 + b]) + P[8 + a] * P[8 + b]) - (a == b ? 1.0 : 0.0)) <= 1e-6;
    for (int k = 0; k < 3; k++) plo[k] = phi[k] = P[4 * k + 3];
    for (int cu = 0; cu < 2; cu++)
        for (int cw = 0; cw < 2; cw++)
        {
            const double qx = ((cu ? (double)c.width : 0.0) - c.cx) / c.fx * R, qy = ((cw ? (double)c.height : 0.0) - c.cy) / c.fy * R;
            for (int k = 0; k < 3; k++)
            {
                const double p = ((P[4 * k] * qx + P[4 * k + 1] * qy) + P[4 * k + 2] * R) + P[4 * k + 3];
                finite = finite && std::isfinite(p);
                plo[k] = std::min(plo[k], p);
                phi[k] = std::max(phi[k], p);
            }
        }
    for (int k = 0; k < 3; k++)
    {
        double lo = P[4 * k + 3] - R, hi = P[4 * k + 3] + R;
        if (finite) lo = std::max(lo, plo[k]), hi = std::min(hi, phi[k]);
        const double a = std::max(std::floor(lo / v) - 1.0 - (double)g.o[k], 0.0);
        const double b = std::min(std::floor(hi / v) + 1.0 - (double)g.o[k], (double)(g.n[k] - 1));
        V.lo[k] = a <= b ? (int)a : 0;
        V.size[k] = a <= b ? (int)(b - a) + 1 : 0;
    }
}

// The control points of n uniform cubic B-splines as the trajectory and heading jobs take them (include/dsm.h):
// offsets[0] = 0, 7 to 256 points per trajectory, at most max_points in all, every coordinate finite
static inline bool spline_points_ok(const double *points, const int32_t *offsets, int n, int max_points)
{
    if (offsets[0] != 0) return false;
    for (int j = 0; j < n; j++)
    {
        if (offsets[j + 1] < offsets[j]) return false;
        const int m = offsets[j + 1] - offsets[j];
        if (m < 7 || m > DSM_TRAJECTORY_MAX_POINTS || offsets[j + 1] > max_points) return false;
    }
    for (size_t c = 0; c < 3 * (size_t)offsets[n]; c++)
        if (!std::isfinite(points[c])) return false;
    return true;
}
