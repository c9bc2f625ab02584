/*
 * dsm.h — C ABI of the H100-native DenseSurfelMapping per-frame hot path.
 *
 * Drop-in boundary: this library replaces exactly one call site of the reference,
 *
 *     SurfelMap::fuse_map -> fusion_functions.fuse_initialize_map(...)   surfel_map.cpp:1066-1073
 *     SurfelMap::SurfelMap -> fusion_functions.initialize(...)            surfel_map.cpp:53
 *
 * i.e. the public surface of `class FusionFunctions` (fusion_functions.h:84-94).  Everything
 * behind it (superpixel extraction, back-projection + normals, robust per-superpixel plane
 * fit, surfel associate / weighted-fuse / initialise; fusion_functions.cpp:30-975) runs as
 * hand-written sm_90a CUDA kernels.  There is NO CPU fallback: every entry point returns
 * DSM_E_CUDA / DSM_E_NODEVICE when no H100-class (sm_90) device is usable.
 *
 * Conventions: extern "C", plain pointers and sizes, int return (0 = DSM_OK, negative = error),
 * no exceptions cross the boundary, one context per GPU, calls on one context are serialised
 * by the caller (the reference is single-threaded at this call site too: ros_node.cpp:38-41).
 * Element layouts are byte-identical to the reference PODs (elements.h:5-31).
 *
 * Numerical contract: superpixel labels and the clustering state (seed x, y, intensity, Huber mean depth, stable flag)
 * are bit-identical to the serialised reference; the plane fit and everything downstream of it (seed normal / position /
 * view_cos / size, surfel geometry) agree within 1e-4 (norm-based) but are NOT bit-identical: their float / fp64 sums are
 * accumulated lane-partially and tree-reduced instead of sequentially (fusion_functions.cpp:117-119, :849-860).  A frame's
 * results do not depend on the batch size, on chunking or on which entry point delivered it: every entry point runs the
 * same kernels.
 *
 * INTEGRATION.md shows the reference-side binding (a FusionFunctions-compatible C++ adapter,
 * include/dsm_fusion_functions.hpp, plus the ctypes stub used by the tests).
 */
#ifndef DSM_H
#define DSM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSM_VERSION 200 /* 0.2.0: tile schedule (TMA-staged kernels), multi-GPU gather in the C ABI, runtime constant sets */

/* ---- error codes ---- */
#define DSM_OK 0
#define DSM_E_INVALID (-1)   /* bad argument (null pointer, negative count, batch too large ...) */
#define DSM_E_SHAPE (-2)     /* unsupported image shape: W%8 > 4 or H%8 > 4 (reference UB, fusion_functions.cpp:408-451) */
#define DSM_E_NODEVICE (-3)  /* no CUDA device / device is not sm_90 */
#define DSM_E_CUDA (-4)      /* a CUDA runtime call or kernel failed; see dsm_last_error() */
#define DSM_E_NOMEM (-5)     /* device or host allocation failed */
#define DSM_E_CAPACITY (-6)  /* more surfels than the context was created for */
#define DSM_E_STATE (-7)     /* call sequence error (e.g. download before run) */
#define DSM_E_NCCL (-8)      /* NCCL unavailable or a collective failed */
#define DSM_E_IO (-9)        /* a file could not be opened, read or written (dsm_write_*, dsm_map_*) */

/* ---- element types: byte-identical to the reference ---- */

/* reference: elements.h:22-31 `struct SurfelElement` (44 bytes) */
typedef struct dsm_surfel_t
{
    float px, py, pz;   /* world position */
    float nx, ny, nz;   /* world normal */
    float size;         /* radius, metres */
    float color;        /* gray 0..255 stored as float */
    float weight;
    int32_t update_times; /* 0 == dead */
    int32_t last_update;  /* reference KEYFRAME index of the last fuse (surfel_map.cpp:145,161) */
} dsm_surfel_t;

/* reference: elements.h:5-20 `struct Superpixel_seed` (60 bytes) — parity/debug readback only */
typedef struct dsm_seed_t
{
    float x, y;
    float size;
    float norm_x, norm_y, norm_z;
    float posi_x, posi_y, posi_z;
    float view_cos;
    float mean_depth;
    float mean_intensity;
    uint8_t fused;
    uint8_t stable;
    uint8_t _pad[2];
    float min_eigen_value; /* debug fields of the reference; always 0 here */
    float max_eigen_value;
} dsm_seed_t;

/* ---- context parameters ---- */
/* The first eight fields are the arguments of FusionFunctions::initialize
 * (fusion_functions.h:84-87, fusion_functions.cpp:7-28).  The rest size the GPU-resident
 * buffers.  SP_SIZE 8, ITERATION_NUM 3 and MAX_ANGLE_COS 0.1 (fusion_functions.h:8-11) are compiled into the kernels;
 * the four constants the reference ships in two sets ("drive" / "RGBD", fusion_functions.h:12-21) are run-time
 * values: a new context holds the drive set, dsm_set_constants() switches. */
typedef struct dsm_params
{
    int32_t width, height;
    float fx, fy, cx, cy;
    float fuse_far, fuse_near;
    int32_t max_batch;         /* frames processed per dsm_batch_* call (>= 1) */
    int32_t max_local_surfels; /* capacity of the local-surfel pool, summed over the batch */
} dsm_params;

typedef struct dsm_ctx dsm_ctx;

/* ---- lifetime ---- */
int dsm_version(void);
const char *dsm_strerror(int code);
/* last CUDA/NCCL error text recorded on this context (never NULL) */
const char *dsm_last_error(const dsm_ctx *ctx);

/* Replaces FusionFunctions::initialize (fusion_functions.cpp:7-28).  `device` is the CUDA
 * ordinal.  `cuda_stream` may be NULL (the context creates its own non-blocking stream) or a
 * cudaStream_t owned by the caller on which all work of this context is enqueued. */
int dsm_create(const dsm_params *params, int device, void *cuda_stream, dsm_ctx **out);
void dsm_destroy(dsm_ctx *ctx);
int dsm_num_seeds(const dsm_ctx *ctx); /* S = (W/8)*(H/8) */

/* The constants the reference selects at compile time by (un)commenting one of two #define blocks (fusion_functions.h:12-21):
 * HUBER_RANGE (Huber-Newton mean depth :540-547, plane-fit inliers :850 and robust weights :134-169), and BASELINE,
 * DISPARITY_ERROR, MIN_TOLERATE_DIFF (depth tolerance of the surfel association :252-253).  Applies to every later call on
 * the context; a fresh context holds DSM_CONSTANTS_DRIVE. */
typedef struct dsm_constants
{
    double huber_range, baseline, disparity_error, min_tolerate_diff;
} dsm_constants;
#define DSM_CONSTANTS_DRIVE {0.4, 0.5, 4.0, 0.1}   /* fusion_functions.h:13-16, the set the reference ships enabled (KITTI) */
#define DSM_CONSTANTS_RGBD {0.05, 0.08, 1.0, 0.05} /* fusion_functions.h:18-21, the commented RGB-D / VINS set */
int dsm_set_constants(dsm_ctx *ctx, const dsm_constants *constants);

/* dsm_batch_run executes a resident batch as `sub_batches` (1..4) groups of frames on concurrent CUDA streams; results do
 * not depend on it (frames are independent).  Default 2: most kernels of the schedule are issue- or latency-bound, two
 * concurrent half-batches fill each other's tails.  1 = the whole batch as one launch sequence (what per-kernel timing
 * with dsm_profile_* should use: concurrent kernels share the SMs and stretch each other's event-pair durations). */
int dsm_set_concurrency(dsm_ctx *ctx, int sub_batches);

/* ---- reference-identical single-frame call ----
 * Replaces FusionFunctions::fuse_initialize_map (fusion_functions.cpp:30-83) with the same
 * semantics: `gray` is CV_8UC1 (row pitch gray_pitch bytes), `depth` CV_32FC1 metres (row
 * pitch depth_pitch bytes), `pose_colmajor` = Eigen::Matrix4f T_world<-cam memory order,
 * `local[n_local]` is updated IN PLACE and never resized (dead surfels are flagged
 * update_times == 0, the caller compacts: surfel_map.cpp:1077-1109), `new_out` receives the
 * newly initialised surfels in seed-index order (the reference clears and push_backs,
 * fusion_functions.cpp:320,359); at most new_cap are written, *n_new is the full count.
 * Host pointers; uploads, runs all kernels, downloads, synchronises.
 * Input domain: depth values are metres, <= 0.01 means "no measurement"; valid depths must be >= 0.02 m
 * (below that the reference itself indexes out of bounds, DESIGN.md 1.3). */
int dsm_fuse_frame(dsm_ctx *ctx, int reference_frame_index,
                   const uint8_t *gray, size_t gray_pitch,
                   const float *depth, size_t depth_pitch,
                   const float pose_colmajor[16],
                   dsm_surfel_t *local, int n_local,
                   dsm_surfel_t *new_out, int new_cap, int *n_new);

/* ---- batch of independent frames (BASELINE configs 3/4) ----
 * Frame b has its own image pair, pose, reference index and its own slice of the local pool:
 * local[local_offsets[b] .. local_offsets[b+1]).  gray/depth are tightly packed
 * [n_frames][H][W].  new_out is [n_frames][S] (S = dsm_num_seeds), n_new is [n_frames].
 * The three stages are exposed separately so that a caller (and bench.py) can keep inputs
 * resident in HBM and time the kernels alone; dsm_fuse_batch() chains them and synchronises. */
int dsm_batch_upload(dsm_ctx *ctx, int n_frames, const int32_t *reference_frame_index,
                     const uint8_t *gray, const float *depth, const float *poses_colmajor,
                     const dsm_surfel_t *local, const int32_t *local_offsets);
int dsm_batch_run(dsm_ctx *ctx);     /* enqueue K0..K6 for the uploaded batch; asynchronous */
int dsm_batch_download(dsm_ctx *ctx, dsm_surfel_t *local_out, dsm_surfel_t *new_out, int32_t *n_new);
int dsm_sync(dsm_ctx *ctx);          /* wait for the context's stream */
int dsm_fuse_batch(dsm_ctx *ctx, int n_frames, const int32_t *reference_frame_index,
                   const uint8_t *gray, const float *depth, const float *poses_colmajor,
                   dsm_surfel_t *local, const int32_t *local_offsets,
                   dsm_surfel_t *new_out, int32_t *n_new);
/* The same call split in two so that a caller can double-buffer: dsm_fuse_batch_async() enqueues the copies
 * and kernels and returns; every host buffer must stay valid and untouched until dsm_batch_wait() returns.
 * One batch per context may be in flight; with two contexts the H2D copies of batch k+1 overlap the kernels
 * of batch k completely (what bench.py's e2e leg does). */
int dsm_fuse_batch_async(dsm_ctx *ctx, int n_frames, const int32_t *reference_frame_index,
                         const uint8_t *gray, const float *depth, const float *poses_colmajor,
                         dsm_surfel_t *local, const int32_t *local_offsets,
                         dsm_surfel_t *new_out, int32_t *n_new);
int dsm_batch_wait(dsm_ctx *ctx);
/* Re-upload only the local pool (the kernels update it in place, so a benchmark that replays
 * the same batch must restore it between steps). Device-to-device from an internal snapshot
 * taken at the last dsm_batch_upload. */
int dsm_batch_restore_pool(dsm_ctx *ctx);

/* ---- GPU-resident pool for a sequential stream (SURVEY.md §8f rows 1-2) ----
 * The pool of ONE stream lives on the device between frames, so per
 * frame only the image pair and the pose cross PCIe.  Semantics mirror what SurfelMap does around
 * the hot-path call:
 *   dsm_pool_upload            local_surfels := given array
 *   dsm_fuse_frame_resident    fuse_initialize_map on the resident pool, THEN the post-step of
 *                              SurfelMap::fuse_map (surfel_map.cpp:1077-1109), in place: new surfels fill the
 *                              dead slots from the highest index down, the rest are appended, leftover dead slots
 *                              take the back element.  The pool equals the reference's local_surfels element for
 *                              element (byte for byte given the same fuse results), and slots are stable: a
 *                              surfel keeps its index until it dies or is the back element moved into a hole.
 *                              *n_new (optional) = number of new surfels; passing it synchronises.  The call is
 *                              dsm_fuse_stream_resident with n_frames = 1, except that image rows lie gray_pitch /
 *                              depth_pitch bytes apart; it is ordered as stated there.
 *   dsm_pool_transform         warp_active_surfels_cpu_kernel (surfel_map.cpp:750-789):
 *                              p <- W p, n <- R_W n for every pool surfel after a loop closure
 *                              (W = T_loop * T_cam^-1 computed by the caller in fp64, cast to f32).
 *   dsm_pool_retire            the removal half of SurfelMap::move_add_surfels (surfel_map.cpp:1479-1497):
 *                              the live surfels whose last_update == keyframe_index are copied out in
 *                              pool order (they become that pose's attached_surfels) and flagged dead
 *                              (update_times = 0; the next fuse post-step recycles their slots, as the reference does).  Counts first: if more than
 *                              `cap` surfels match, nothing is flagged, *n_out is the number needed and the call
 *                              returns DSM_E_CAPACITY.  Synchronises.
 *   dsm_pool_append            the insertion half (surfel_map.cpp:1583-1587): surfels of poses that
 *                              re-enter the drift-free set are appended to the pool.  Synchronises.
 *   dsm_pool_size / dsm_pool_download   read back (synchronise). */
int dsm_pool_upload(dsm_ctx *ctx, const dsm_surfel_t *local, int n_local);
int dsm_fuse_frame_resident(dsm_ctx *ctx, int reference_frame_index,
                            const uint8_t *gray, size_t gray_pitch, const float *depth, size_t depth_pitch,
                            const float pose_colmajor[16], int *n_new);
/* n consecutive frames of the SAME stream in one call (tightly packed [n][H][W] images, [n][16] poses): results are
 * those of n calls of dsm_fuse_frame_resident (same kernels, same order on the pool), but the pose- and pool-independent stages (superpixels, normals, plane fit) of all n frames run as one
 * batch; only fuse / initialise / post-step run frame by frame.  Trades
 * n-1 frames of latency for throughput (offline sequences, or a node that lags behind its camera).  n <= max_batch;
 * with 2n <= max_batch consecutive runs use alternate halves of the frame slots: the copy and the batched stages of one
 * run overlap the frame-by-frame stages of the previous one.  n_new (optional, [n]) = new surfels per frame; passing it
 * synchronises.
 * Ordering of the resident stream calls (this one, dsm_fuse_frame_resident and dsm_fuse_stream_window): a run's
 * frame-by-frame stages follow everything enqueued on the context's stream before the call, and work enqueued on that
 * stream after the call follows them.  Its batched stages rewrite the frame slots of the run's staging half, new surfels
 * and counts included (DSM_BUF_NEW_SURFELS / DSM_BUF_NEW_COUNTS), and wait only for what was enqueued on the context's
 * stream before the PREVIOUS call began.  With alternating halves that is the last run on the same half and every read
 * of its slots enqueued before the next call; a read enqueued later may see the slots rewritten.  The same holds for
 * batch calls (dsm_batch_upload / _run / _download) enqueued between two resident calls: they use frame slots from 0
 * and are not ordered before the batched stages of the call after the next.  The host waits for the same point before
 * it reuses a half's staging buffers, so it blocks when it gets more than two calls ahead.  With a single half
 * (2n > max_batch, e.g. every single-frame call at max_batch = 1) the run is ordered on the context's stream like
 * every other call, and the host waits at its entry for everything enqueued on that stream before it.  The resident
 * stream calls return DSM_E_STATE while a dsm_fuse_batch_async batch is in flight. */
int dsm_fuse_stream_resident(dsm_ctx *ctx, int n_frames, const int32_t *reference_frame_index,
                             const uint8_t *gray, const float *depth, const float *poses_colmajor, int32_t *n_new);
int dsm_pool_transform(dsm_ctx *ctx, const float W_colmajor[16]);
int dsm_pool_retire(dsm_ctx *ctx, int keyframe_index, dsm_surfel_t *out, int cap, int *n_out);
int dsm_pool_append(dsm_ctx *ctx, const dsm_surfel_t *surfels, int n);
int dsm_pool_size(dsm_ctx *ctx, int *n_local);
int dsm_pool_download(dsm_ctx *ctx, dsm_surfel_t *out, int cap, int *n_local);

/* ---- output side: point clouds and files (SURVEY.md §8f row 4) ----
 * pcl::PointXYZI as the reference publishes and saves it, without PCL's SSE padding: 16 bytes. */
typedef struct dsm_point_t
{
    float x, y, z;
    float intensity; /* SurfelElement::color, gray 0-255 */
} dsm_point_t;
/*   dsm_pool_export_cloud      the cloud builders of SurfelMap over local_surfels: every pool surfel with
 *                              update_times >= min_update_times becomes one point {px, py, pz, color}, in pool
 *                              order like the serial push_back loops.  min_update_times = 5:
 *                              publish_active_pointcloud (surfel_map.cpp:1398-1417), the local part of
 *                              publish_all_pointcloud (:1419-1454) and save_cloud (:1153-1173); = 1: the local part
 *                              of publish_neighbor_pointcloud (:1284-1300, "update_times == 0 -> skip").  Filter and
 *                              compaction run on the device; only the selected 16-byte points cross PCIe.
 *                              *n_out = number selected (may exceed cap; min(cap, *n_out) points are written).
 *   dsm_pool_export_surfels    the same selection returning whole surfels (what save_mesh iterates, :1241-1247).
 *   Both synchronise and leave the pool untouched.
 *   dsm_write_pcd              pcl::io::savePCDFile(name, cloud) of surfel_map.cpp:1171 (PCD v0.7, fields
 *                              x y z intensity; binary = 0 is what the reference writes).  Host only.
 *   dsm_write_ply_mesh         SurfelMap::save_mesh (:1229-1280): one hexagon (6 vertices, 4 triangles) per
 *                              surfel via push_a_surfel (:1175-1226), ASCII PLY.  The caller passes the attached
 *                              surfels of every pose followed by dsm_pool_export_surfels(ctx, 5, ...).  Host only.
 *   dsm_mesh_vertices          push_a_surfel alone: 36 floats (6 x {x, y, z, c, c, c}) per surfel.
 *   dsm_frame_raw_cloud        publish_raw_pointcloud (:1115-1151) on the context's copy of a frame: every pixel
 *                              back-projected into the world, holes included (depth 0 -> T), W*H points in the
 *                              reference's column-major loop order (point k = i*H + j for column i, row j), intensity =
 *                              gray.  pose7 = geometry_msgs::Pose {px, py, pz, qx, qy, qz, qw}: R =
 *                              Quaternionf((float)qw, (float)qx, (float)qy, (float)qz).toRotationMatrix() (not
 *                              normalised), T = (float)position; the points are bit-identical to the reference's float
 *                              loop.  `frame` indexes the frames of the context's most recent call that took images:
 *                              dsm_fuse_frame / dsm_fuse_frame_resident -> 0, dsm_fuse_stream_resident -> 0..n-1,
 *                              dsm_batch_upload / dsm_fuse_batch[_async] -> 0..n_frames-1 (an asynchronous batch is
 *                              waited for).  DSM_E_STATE before any such call, DSM_E_INVALID for a frame outside it.
 *                              *n_out = W*H, min(cap, W*H) points are written.  Synchronises; touches no pool, label or
 *                              seed state.  The first call allocates W*H*16 bytes of device memory, kept with the context.
 *   The neighbourhood cloud of publish_neighbor_pointcloud (:1283-1383) is dsm_pool_export_cloud(ctx, 1, ...) followed by
 *   dsm_inactive_export_poses(ctx, get_driftfree_poses(reference_index, 2*drift_free_poses), ...) (inactive store below). */
int dsm_pool_export_cloud(dsm_ctx *ctx, int min_update_times, dsm_point_t *out, int cap, int *n_out);
int dsm_pool_export_surfels(dsm_ctx *ctx, int min_update_times, dsm_surfel_t *out, int cap, int *n_out);
int dsm_write_pcd(const char *path, const dsm_point_t *points, size_t n, int binary);
int dsm_write_ply_mesh(const char *path, const dsm_surfel_t *surfels, size_t n);
int dsm_mesh_vertices(const dsm_surfel_t *surfels, size_t n, float *vertices36);
int dsm_frame_raw_cloud(dsm_ctx *ctx, int frame, const double pose7[7], dsm_point_t *out, int cap, int *n_out);

/* ---- superpixel normal image of a frame: FusionFunctions::debug_show (fusion_functions.cpp:977-1006) ----
 * The reference's one view of what the superpixel stage did, built on the device from the labels and plane fits the
 * context already holds (3 B/px cross PCIe instead of the 4 B/px labels plus 60 B per seed of dsm_get_labels /
 * dsm_get_seeds).  bgr receives H rows of 3*W bytes at a row pitch of `pitch` bytes (a cv::Mat of CV_8UC3):
 *   pixel (x, y) = {b0, b1, b2} = {|norm_x|, |norm_y|, |norm_z|} * 255 of the seed that labels it (cv::Vec3b order,
 *   :986-988); {0, 0, 0} when x + 1 < W and the label of (x+1, y) differs, or y + 1 < H and the label of (x, y+1)
 *   differs (:991-1000).  A seed whose plane fit was rejected has a zero normal, so its superpixel is black.
 * Each channel is the reference's arithmetic: (double)fabs(n) * 255 (exact in double), converted to uchar the way its
 * x86-64 build does, through a truncating 32-bit conversion whose low byte is kept.  A NaN normal (DESIGN.md 1.3:
 * a superpixel whose pixel normals are all zero) gives 0; for |n| <= 1 the byte is floor(|n| * 255).
 * Exactness: given the context's own labels and seeds (dsm_get_labels / dsm_get_seeds of the same frame slot), the image
 * equals the reference's debug_show byte for byte.  Against the reference's whole pipeline the black boundary pixels
 * are exact (labels are bit-identical) and a colour differs by at most 1 per channel, in the rare superpixel whose
 * |n| * 255 lies within the 1e-4 plane-normal budget of an integer.
 * `frame` as in dsm_frame_raw_cloud: the frame-th frame of the most recent call that took images (an asynchronous
 * batch is waited for).  DSM_E_STATE before any such call, or when that call's schedule has not run through the plane
 * fit (dsm_batch_upload without dsm_batch_run, or a run cut short by dsm_debug_stop_after before the plane fit);
 * DSM_E_INVALID for a frame outside the call, a null bgr or pitch < 3*W.  Bytes between 3*W and pitch are left
 * untouched.  Synchronises; touches no pool, label, seed or inactive-store state.  The first call allocates
 * H * 3*Wp bytes (Wp = W rounded up to 16) of device memory, kept with the context. */
int dsm_frame_superpixel_image(dsm_ctx *ctx, int frame, uint8_t *bgr, size_t pitch);

/* ---- inactive store ----
 * What SurfelMap keeps per pose outside the drift-free window -- PoseElement::attached_surfels and the mirror
 * inactive_pointcloud (surfel_map.h:36-46) -- resident on the device next to the local pool, so that
 * move_add_surfels and the loop-closure warp of the inactive surfels never cross PCIe.  Segments are kept dense in
 * retirement order; the segment table lives on the device, where retirements and reactivations update it (the calls
 * below and dsm_fuse_stream_window), and the calls below that synchronise refresh a host mirror of it.
 *   dsm_inactive_reserve      capacity in surfels (once, while the store is empty)
 *   dsm_inactive_retire       move_add_surfels removal loop (surfel_map.cpp:1479-1497): local surfels with
 *                             update_times > 0 and last_update == keyframe_index become that pose's segment (pool
 *                             order) and are flagged dead in the pool.  Synchronises; *n_moved optional.
 *   dsm_inactive_reactivate   insertion (surfel_map.cpp:1583-1587): the pose's segment returns to the end of the pool
 *   dsm_inactive_transform    warp_inactive_surfels_cpu_kernel for one pose (surfel_map.cpp:704-733), asynchronous
 *   dsm_inactive_export_cloud inactive_pointcloud as the node publishes / saves it (store order)
 *   dsm_inactive_export_poses the inactive half of publish_neighbor_pointcloud (surfel_map.cpp:1306-1321): the stored
 *                             points of each listed keyframe, concatenated in list order (store order within a keyframe).
 *                             A keyframe with nothing stored contributes nothing -- the reference's skip of local poses
 *                             and of empty attached_surfels (:1311-1316) -- so the caller passes the drift-free BFS list
 *                             of 2*drift_free_poses unchanged.  cap / *n_out as dsm_inactive_export_cloud.
 *                             Both exports return the points as the store holds them, i.e. after dsm_inactive_transform
 *                             every point of a pose is warped; the reference's slice of inactive_pointcloud keeps its last
 *                             point stale (the std::copy(&front, &back) off-by-one of surfel_map.cpp:742, SURVEY.md §8f row 1).
 *   dsm_inactive_download     attached_surfels of one pose (keyframe_index >= 0) or of all poses (< 0; save_mesh)
 *   dsm_inactive_size         surfels / segments currently stored */
int dsm_inactive_reserve(dsm_ctx *ctx, int max_inactive_surfels);
int dsm_inactive_retire(dsm_ctx *ctx, int keyframe_index, int *n_moved);
int dsm_inactive_reactivate(dsm_ctx *ctx, int keyframe_index, int *n_moved);
int dsm_inactive_transform(dsm_ctx *ctx, int keyframe_index, const float W_colmajor[16]);
int dsm_inactive_export_cloud(dsm_ctx *ctx, dsm_point_t *out, int cap, int *n_out);
int dsm_inactive_export_poses(dsm_ctx *ctx, const int32_t *keyframes, int n_keyframes, dsm_point_t *out, int cap, int *n_out);
int dsm_inactive_download(dsm_ctx *ctx, int keyframe_index, dsm_surfel_t *out, int cap, int *n_out);
int dsm_inactive_size(dsm_ctx *ctx, int *n_surfels, int *n_segments);

/* ---- checkpoint and resume of the GPU-resident map (DESIGN.md §8.4) ----
 * Between frames the pool, the inactive store and its segment table are the whole device state of a map, so a drive
 * resumed from a checkpoint is byte-identical to the same drive run without interruption.
 *   dsm_inactive_segments  the segment table in store order: kf_ofs_cnt[i] = (keyframe, offset, count) of segment i.
 *                          min(cap, n) entries written, *n_out = n.  Synchronises (reports a rejected frame as every
 *                          synchronising reader does).  DSM_E_STATE without dsm_inactive_reserve.
 *   dsm_inactive_load      replaces the store's contents and table.  Checked on the host, in this order, before the device
 *                          is touched, so a failure leaves the store as it was: DSM_E_STATE without a reservation or while
 *                          a publish snapshot is in flight; DSM_E_CAPACITY for n above the reservation; DSM_E_INVALID for a
 *                          malformed table (offsets not contiguous from 0, a count below 1, counts not summing to n, a
 *                          negative keyframe) and for a surfel with update_times == 0 or a last_update other than its
 *                          segment's keyframe (true of every store the library builds).  A keyframe may own several
 *                          segments.  With publishing enabled the next snapshot reports inactive_changed_from = 0 and
 *                          forwards every chunk, as after dsm_inactive_reserve.  Synchronises.
 *   dsm_map_save           writes the pool (slot order), the store (store order), the table and the caller's `extra` bytes
 *                          (opaque to the library) to one versioned little-endian file with a 64-bit checksum, together
 *                          with the context's geometry and constants.  Needs a resident pool (DSM_E_STATE); a store is
 *                          optional.  A synchronising reader: a pending rejected frame is reported as DSM_E_CAPACITY and
 *                          cleared, and no file is written; the next save writes the map of the last applied frame.  The
 *                          file is written under a temporary name in the same directory, flushed to the disk and renamed:
 *                          DSM_E_IO on any I/O failure, with nothing left under `path`.
 *   dsm_map_load           reads and checks the whole file before the device is touched, so every failure leaves the map
 *                          as it was: DSM_E_IO if it cannot be read, is truncated or fails its checksum; DSM_E_INVALID for a
 *                          wrong magic or format version, and for geometry or constants other than the context's (set the
 *                          constants before loading; max_batch and the capacities may differ); DSM_E_CAPACITY if the pool
 *                          does not fit max_local_surfels; DSM_E_STATE while a publish snapshot is in flight, or if the file
 *                          has stored surfels and the context no store; then dsm_inactive_load's checks; DSM_E_CAPACITY if
 *                          extra_cap is below the extra section, with *extra_bytes (optional) set and nothing loaded.  Then
 *                          the pool is uploaded (dsm_pool_upload) and the store replaced (dsm_inactive_load; an empty
 *                          store section empties a reserved store).  A checkpoint holds no frame: dsm_frame_raw_cloud and
 *                          dsm_frame_superpixel_image still refer to the most recent call that took images.
 *   dsm_map_peek           the extra section and the segment table of a checkpoint file, checked as dsm_map_load checks
 *                          the file itself (DSM_E_IO / DSM_E_INVALID), without a context: a caller can decide on the file
 *                          before it touches its map.  min(cap, size) of each is written; *extra_bytes and *n_segments
 *                          (optional) receive the sizes. */
int dsm_inactive_segments(dsm_ctx *ctx, int32_t *kf_ofs_cnt /* [cap][3] */, int cap, int *n_out);
int dsm_inactive_load(dsm_ctx *ctx, const dsm_surfel_t *surfels, int n, const int32_t *kf_ofs_cnt, int n_segments);
int dsm_map_save(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes);
int dsm_map_load(dsm_ctx *ctx, const char *path, void *extra, size_t extra_cap, size_t *extra_bytes);
int dsm_map_peek(const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt, int seg_cap,
                 int *n_segments);

/* ---- the node's whole per-frame sequence on the device: move_add_surfels + fuse_map (surfel_map.cpp:154-161) ----
 * dsm_fuse_stream_window is dsm_fuse_stream_resident with each frame's drift-free window step in front of its fuse.
 * For frame t, in order:
 *   1. every keyframe of retire_kf[retire_ofs[t] .. retire_ofs[t+1]) is retired, in list order (= dsm_inactive_retire)
 *   2. every keyframe of reactivate_kf[reactivate_ofs[t] .. reactivate_ofs[t+1]) is reactivated, in list order
 *      (= dsm_inactive_reactivate)
 *   3. frame t is fused on the resident pool, post-step included (= dsm_fuse_frame_resident)
 * The lists are the node's poses_to_remove / poses_to_add of get_add_remove_poses (surfel_map.cpp:1597-1641), which the
 * caller knows before any kernel runs.  Afterwards the pool, the store (contents and order) and its segment list are
 * byte-identical to what that sequence of calls leaves.  Phase 1 (superpixels, plane fits) runs batched and overlaps the
 * previous call exactly as in dsm_fuse_stream_resident; the window step of a frame runs right before its fuse on the
 * same high-priority stream.  All lists empty: the result of dsm_fuse_stream_resident.  n_frames = 1: the single-frame
 * node.  A NULL offset array means empty lists for every frame.
 * Nothing waits for the device unless n_new ([n_frames], optional) is passed: the surfel counts stay on the device.
 * Checked on the host before anything is enqueued:
 *   DSM_E_INVALID  offsets that decrease, more than DSM_WINDOW_MAX_KEYS keys in one frame's list, a negative keyframe,
 *                  a keyframe listed twice in one frame's lists or in both lists of one frame
 *   DSM_E_STATE    a non-empty list without dsm_inactive_reserve, and the errors of dsm_fuse_stream_resident
 * Capacity is checked on the device, with the exact counts, for each frame before any of it is applied: the store after
 * its retirements must fit the reservation, and the pool after its reactivations plus one frame of new surfels (S =
 * dsm_num_seeds) must fit max_local_surfels (the test of dsm_fuse_frame_resident).  A frame that does not fit is not
 * applied, and neither is any later frame, of this call or of later calls: it sets a sticky error word on the device,
 * every resident kernel exits at once while the word is set, and the pool and store stay exactly as after the last
 * applied frame.  The error is returned as DSM_E_CAPACITY by this call when n_new is passed (n_new[t] = -1 for every
 * frame not applied), otherwise by the next call that synchronises with the resident state (dsm_pool_size,
 * dsm_pool_download, dsm_pool_retire, dsm_pool_export_*, dsm_pool_append, dsm_inactive_* except _transform, and the
 * fuse calls that return n_new).  That call clears the word and does nothing else; the map can be read and the stream
 * resumed from the last applied frame.  The segment table has one entry per surfel of the reservation, so it cannot
 * overflow on its own. */
#define DSM_WINDOW_MAX_KEYS 128
int dsm_fuse_stream_window(dsm_ctx *ctx, int n_frames, const int32_t *reference_frame_index,
                           const uint8_t *gray, const float *depth, const float *poses_colmajor,
                           const int32_t *retire_kf, const int32_t *retire_ofs,         /* [n_frames + 1] */
                           const int32_t *reactivate_kf, const int32_t *reactivate_ofs, /* [n_frames + 1] */
                           int32_t *n_new);

/* ---- publishing from inside the stream: the node's active and inactive clouds after a fused frame ----
 * What synchronize_msgs publishes after every fuse (surfel_map.cpp:191-198), enqueued in stream order like a fuse, with
 * one wait (or none, one frame late) and only the changed part of the inactive cloud crossing PCIe.
 *   dsm_publish_enable    once, on a context with a resident pool (DSM_E_STATE otherwise, and when called twice):
 *                         allocates pinned host buffers the device writes directly -- max_local_surfels points for the
 *                         active cloud and, with a store, its reservation for the inactive cloud -- plus a device shadow
 *                         of the inactive cloud as the host last received it (16 B per reserved surfel).  DSM_E_NOMEM.
 *                         A later dsm_inactive_reserve rebuilds the inactive buffers with the store (DSM_E_STATE while a
 *                         snapshot is in flight).
 *   dsm_publish_enqueue   asynchronous, ordered on the context's stream exactly like dsm_pool_transform: the snapshot is
 *                         the map after everything enqueued before it (the frame-by-frame stages of the preceding
 *                         resident call included) and before anything enqueued after it.  Runs the ordered selection of
 *                         dsm_pool_export_cloud(min_update_times) into the active buffer and one pass over the store that
 *                         compares each chunk of 256 points with the shadow and forwards the chunks that differ.  Never
 *                         waits and reads nothing back.  DSM_E_STATE before dsm_publish_enable, and while a snapshot is
 *                         enqueued and not yet waited for (the host may be reading the buffers).
 *   dsm_publish_wait      waits for that snapshot only, not for the stream.  *active / *inactive are the context's pinned
 *                         buffers: valid until the next dsm_publish_enqueue (or dsm_inactive_reserve), never to be freed
 *                         or written.  active[0 .. *n_active) is what dsm_pool_export_cloud(ctx, min_update_times, ...)
 *                         would have returned at the snapshot's position in the stream, inactive[0 .. *n_inactive) what
 *                         dsm_inactive_export_cloud would have, byte for byte (no store: 0 points, *inactive NULL).
 *                         Points below *inactive_changed_from are bit-identical to the previous snapshot's: it is the
 *                         lowest index whose point differs from the previous snapshot, an index at or beyond the previous
 *                         size counting as different, and *n_inactive when there is none.  The first snapshot, and the
 *                         first after dsm_inactive_reserve, report 0.  Any out-pointer may be NULL.  If a frame of
 *                         dsm_fuse_stream_window had been rejected before the snapshot, the call returns DSM_E_CAPACITY
 *                         with the clouds of the last applied frame and does NOT clear the error: the next synchronising
 *                         call reports and clears it as stated above.  DSM_E_STATE with no snapshot enqueued.
 *   dsm_debug_publish_chunks   the number of 256-point chunks the last waited snapshot forwarded to the host (0 when the
 *                         store did not change); DSM_E_STATE while a snapshot is in flight. */
int dsm_publish_enable(dsm_ctx *ctx);
int dsm_publish_enqueue(dsm_ctx *ctx, int min_update_times);
int dsm_publish_wait(dsm_ctx *ctx, const dsm_point_t **active, int *n_active, const dsm_point_t **inactive, int *n_inactive,
                     int *inactive_changed_from);
int dsm_debug_publish_chunks(dsm_ctx *ctx, int *count);

/* ---- the map as a distance field for planners (DESIGN.md §8.7) ----
 * A local voxel grid of the resident map and its exact Euclidean distance transform, built in stream order like a publish
 * snapshot, so that it follows every loop closure the map follows.  Grid: voxel edge v, size (nx, ny, nz).  A request
 * centred on c has the integer origin o_k = floor(c_k / (double)v) - floor(n_k / 2).  Its obstacle points are those of
 * dsm_pool_export_cloud(min_update_times) and dsm_inactive_export_cloud at the request's position in the stream; a point p
 * marks voxel q - o, q_k = floorf(p_k / v) in fp32, when o_k <= q_k < o_k + n_k on every axis (compared in fp32; a NaN
 * or infinite coordinate marks nothing).  dist[(z * ny + y) * nx + x] = sqrtf((float)d2) * v, d2 the smallest squared
 * integer distance from voxel (x, y, z) to an occupied voxel (0 on one), +INFINITY everywhere when none is occupied.
 * Unsigned: every voxel without an obstacle point counts as free (dsm_field_enqueue_known, below, measures the distance to
 * anything not known to be free).
 *   dsm_field_enable    once, on a context with a resident pool (DSM_E_STATE otherwise, and when called twice).  v finite
 *                       and > 0, each size in [1, 1024] (DSM_E_INVALID).  Allocates the occupancy grid (1 B per voxel)
 *                       and the distance grid (4 B per voxel) on the device, a pinned host copy of the distance grid and
 *                       an event.  DSM_E_NOMEM, with nothing kept.
 *   dsm_field_enqueue   asynchronous, ordered on the context's stream exactly like dsm_publish_enqueue; never waits and
 *                       reads nothing back.  DSM_E_INVALID for min_update_times < 1, a non-finite centre, or an origin with
 *                       |o_k| or |o_k + n_k| above 2^24; DSM_E_STATE before dsm_field_enable, and while a field is
 *                       enqueued and not yet waited for.
 *   dsm_field_wait      waits for that field only.  *dist is the context's pinned buffer of nx * ny * nz floats, valid
 *                       until the next dsm_field_enqueue, never to be freed or written; origin receives o and
 *                       *n_occupied the number of occupied voxels.  Any out-pointer may be NULL.  If a frame of
 *                       dsm_fuse_stream_window had been rejected before the request, returns DSM_E_CAPACITY with the
 *                       field of the last applied frame and does NOT clear the error, as dsm_publish_wait.  DSM_E_STATE
 *                       with no field enqueued.
 * dsm_inactive_reserve, dsm_inactive_load, dsm_map_load and dsm_map_load_journal return DSM_E_STATE while a field is in
 * flight. */
typedef struct dsm_field_params
{
    float voxel;
    int32_t nx, ny, nz;
} dsm_field_params;
int dsm_field_enable(dsm_ctx *ctx, const dsm_field_params *params);
int dsm_field_enqueue(dsm_ctx *ctx, const double center[3], int min_update_times);
int dsm_field_wait(dsm_ctx *ctx, const float **dist, int32_t origin[3], int *n_occupied);
/* dsm_field_enqueue_resident: dsm_field_enqueue (same checks, ordering, kernels and grid) that copies only the header
 * words to the host; the grid stays on the device for dsm_field_query_*.  dsm_field_wait on such a request returns
 * *dist = NULL with the same origin, n_occupied and DSM_E_CAPACITY contract. */
int dsm_field_enqueue_resident(dsm_ctx *ctx, const double center[3], int min_update_times);

/* ---- planner queries against the latest distance field, on the device (DESIGN.md §8.8) ----
 * A query reads the grid of the latest field request (any enqueue call, waited for or not), in stream order behind
 * it, with that request's origin o and voxel edge v captured at the query's enqueue; a later field request may be
 * enqueued while a query is in flight and does not change what the query reads.  Only the grid is read, never the map.
 *
 * Point query (fp64 addressing, fp32 arithmetic; voxel x covers [(o + x) v, (o + x + 1) v), its value at the centre).
 * Per axis k: u_k = p_k / (double)v - (double)o_k - 0.5 in fp64.  The point is inside when 0 <= u_k <= n_k - 1 on every
 * axis (fp64 compares, NaN fails); then i_k = min(floor(u_k), max(n_k - 2, 0)), j_k = min(i_k + 1, n_k - 1) and
 * t_k = (float)(u_k - i_k).  With lerp(a, b, t) = a + t * (b - a) in fp32 (one rounding per operation) and c_xyz the
 * corner taking i or j per axis (c100 takes j on x):
 *   dist = lerp(lerp(lerp(c000, c100, tx), lerp(c010, c110, tx), ty), lerp(lerp(c001, c101, tx), lerp(c011, c111, tx), ty), tz)
 *   gx   = lerp(lerp(c100 - c000, c110 - c010, ty), lerp(c101 - c001, c111 - c011, ty), tz) / v
 *   gy   = lerp(lerp(c010 - c000, c110 - c100, tx), lerp(c011 - c001, c111 - c101, tx), tz) / v
 *   gz   = lerp(lerp(c001 - c000, c101 - c100, tx), lerp(c011 - c010, c111 - c110, tx), ty) / v
 * Outside: dist is the canonical quiet NaN (unknown, not free) and the gradient 0.  A field with no occupied voxel (a
 * known field: with every voxel free) gives every inside point dist = +INFINITY and a zero gradient.
 *
 * Trajectory clearance.  Trajectory j is the polyline of waypoints offsets[j] .. offsets[j + 1] - 1, sampled in fp64:
 * each segment a -> b with L = sqrt((dx^2 + dy^2) + dz^2) and m = max(1, ceil(L / (double)step)) (counted on the host)
 * gives the samples a + ((double)s / m) * (b - a), s in [0, m); the last waypoint is sampled once at the end.  Samples
 * are numbered along the trajectory from 0; each is a point query (distance only).  Per trajectory: min_dist the minimum
 * dist over the inside samples (+INFINITY when none is inside), argmin the lowest sample index attaining it (-1),
 * first_hit the lowest index of an inside sample with dist < radius (-1 when none), n_outside the samples outside.
 *
 *   dsm_field_query_enable   once, after dsm_field_enable (DSM_E_STATE otherwise).  Allocates, for these capacities, one
 *                            packed pinned request buffer and its device twin, one packed device result buffer and its
 *                            pinned copy, and an event.  DSM_E_INVALID for a negative capacity or one above 2^26;
 *                            DSM_E_NOMEM with nothing kept.
 *   dsm_field_query_enqueue  stages points (n_points x 3 doubles), waypoints and offsets (n_trajectories + 1 ints) into
 *                            pinned memory on the calling thread, then enqueues one H2D copy, the kernels, one D2H copy
 *                            of the results and the event on the context's stream; never waits.  A pointer may be NULL
 *                            when its count is 0.  DSM_E_STATE before dsm_field_query_enable, before any field request
 *                            and while a query is in flight.  DSM_E_INVALID for a negative count or one over capacity
 *                            (offsets[n_trajectories] counts the waypoints), offsets[0] != 0 or offsets that do not rise
 *                            strictly, a non-finite waypoint, a step that is not finite and > 0, a radius that is not
 *                            finite and >= 0, or more than 2^26 trajectory samples in the call (this bounds the work of
 *                            one call).  Points may be anything: a NaN or infinite point is outside.
 *   dsm_field_query_wait     waits for that query only.  *samples (n_points) and *clearance (n_trajectories) are the
 *                            context's pinned result arrays, valid until the next dsm_field_query_enqueue; either
 *                            out-pointer may be NULL.  If the field the query read was taken after a rejected frame,
 *                            returns DSM_E_CAPACITY with valid results and does NOT clear the error, as dsm_field_wait.
 *                            DSM_E_STATE with no query enqueued. */
typedef struct dsm_field_sample_t
{
    float dist, gx, gy, gz; /* metres, per metre */
} dsm_field_sample_t;
typedef struct dsm_clearance_t
{
    float min_dist;
    int32_t argmin, first_hit, n_outside;
} dsm_clearance_t;
#define DSM_FIELD_QUERY_MAX_SAMPLES (1 << 26)
int dsm_field_query_enable(dsm_ctx *ctx, int max_points, int max_trajectories, int max_waypoints);
int dsm_field_query_enqueue(dsm_ctx *ctx, const double *points, int n_points, const double *waypoints, const int32_t *offsets,
                            int n_trajectories, float step, float radius);
int dsm_field_query_wait(dsm_ctx *ctx, const dsm_field_sample_t **samples, const dsm_clearance_t **clearance);

/* ---- free versus unknown space: the distance to anything not known to be free (DESIGN.md §8.9) ----
 * The field of dsm_field_enqueue counts every voxel without an obstacle point as free, including space no camera has
 * seen.  A known request carves the voxels the captured views have observed as free with their rays and measures the
 * distance to the nearest voxel NOT known to be free (unknown is an obstacle).  Rays are kept in camera coordinates, one
 * set per captured frame, and every request takes each view's current world pose, so the field follows loop closures.
 *
 * Rays.  dsm_views_capture stores, in seed index order, the fp32 camera-space plane-fit point posi of every seed of the
 * frame with mean_depth > 0 and three finite coordinates (the posi and mean_depth of dsm_get_seeds); other seeds give no
 * ray.  Adjacent rays are one superpixel apart, so beyond the range where that spacing exceeds a voxel some free voxels
 * between rays stay unknown, which is the safe side.
 *
 * Definition (every step fp64, one rounding per operation).  Occupancy is that of dsm_field_enqueue: state 1.  For view j
 * with pose [R | t] (poses[12 j ..], row-major, camera to world) and each ray p of slot slots[j] (widened to fp64):
 *   a = t;  b_k = ((R_k0 p_x + R_k1 p_y) + R_k2 p_z) + t_k;  d = b - a;  L = sqrt((d_0^2 + d_1^2) + d_2^2);
 *   L > (double)max_range: b_k = a_k + ((double)max_range / L) d_k, and the ray is truncated.
 * Traversal (Amanatides-Woo) in voxel units: w_a = a / (double)v, w_b = b / (double)v, i = floor(w_a), e = floor(w_b),
 * delta = w_b - w_a; per axis s_k = sign(delta_k), tD_k = 1 / |delta_k|, tM_k = ((i_k + 1) - w_a_k) / delta_k for
 * delta_k > 0 and (i_k - w_a_k) / delta_k for delta_k < 0, both +inf for delta_k = 0.  Loop: visit i; stop if i == e;
 * k = argmin tM (the lowest axis on ties); stop if tM_k > 1; i_k += s_k, tM_k += tD_k.
 * Carving: a visited voxel with o <= i < o + n becomes free (state 2) unless it is occupied; e of a ray that was not
 * truncated holds the surface and is never carved.  Every other voxel is unknown (state 0).  (A ray whose endpoints
 * overflow to a non-finite value carves nothing.)
 * Distance: dist = sqrtf((float)d2) * v, d2 the smallest squared integer distance to a voxel of state 0 or 1; +INFINITY
 * everywhere when every voxel is free.  With n_views = 0 every voxel that is not occupied is unknown and dist is 0
 * everywhere.  The known distance never exceeds dsm_field_enqueue's distance of the same request.
 *
 *   dsm_views_enable         once, after dsm_field_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID
 *                            unless 1 <= max_views <= DSM_VIEWS_MAX and max_range is finite, > 0 and <= 1024 v (which
 *                            bounds the voxels one ray visits), or when max_views x ceil(S / 128) reaches 2^31 (frames
 *                            of billions of pixels).  Allocates 16 B per ray for max_views x S rays on the
 *                            device, a pinned copy of the state grid (1 B per voxel) and the pinned and device staging
 *                            of max_views poses.  DSM_E_NOMEM with nothing kept.
 *   dsm_views_capture        asynchronous on the context's stream, never waits: overwrites slot `slot` with the rays of
 *                            frame `frame` of the most recent call that took images (as dsm_frame_superpixel_image:
 *                            DSM_E_STATE with no such call or one whose schedule did not run through the plane fit,
 *                            DSM_E_INVALID for a frame outside it).  A frame whose fuse was rejected may be captured.
 *                            DSM_E_INVALID for a slot outside [0, max_views); DSM_E_STATE before dsm_views_enable.
 *   dsm_field_enqueue_known  dsm_field_enqueue's request (same checks, origin, ordering and DSM_E_CAPACITY rule at
 *                            dsm_field_wait) over the views slots[0 .. n_views) at poses (n_views x 12 doubles),
 *                            staged into pinned memory on the calling thread and copied with one H2D copy.  host_copy =
 *                            0 keeps both grids on the device, as dsm_field_enqueue_resident.  DSM_E_STATE before
 *                            dsm_views_enable; DSM_E_INVALID for n_views < 0 or > max_views, a slot out of range or never
 *                            captured, or a non-finite pose entry.  Queries (dsm_field_query_*) read its distance grid
 *                            like any other field's.
 *   dsm_field_state          the state grid [z][y][x] of the last waited known request (pinned, valid until the next
 *                            field enqueue; NULL for host_copy = 0) and its number of free voxels.  DSM_E_STATE when the
 *                            last waited request was not a known one.  dsm_field_wait returns a known request's dist,
 *                            origin and n_occupied as any other's. */
#define DSM_VIEWS_MAX 65536
int dsm_views_enable(dsm_ctx *ctx, int max_views, float max_range);
int dsm_views_capture(dsm_ctx *ctx, int frame, int slot);
int dsm_field_enqueue_known(dsm_ctx *ctx, const double center[3], int min_update_times, const int32_t *slots, const double *poses,
                            int n_views, int host_copy);
int dsm_field_state(dsm_ctx *ctx, const uint8_t **state, int *n_free);

/* ---- views in the checkpoint: resume known space (DESIGN.md §8.18) ----
 * Without this call, checkpoints carry no views and a load leaves the slot table empty, so every known request after a
 * restart carves nothing.  With it, every checkpoint of the context (dsm_map_save, dsm_checkpoint_enqueue, both kinds of
 * dsm_checkpoint_enqueue_incremental) carries the ascending list of filled slots and, for each, its S = dsm_num_seeds
 * rays exactly as dsm_views_capture wrote them (float4, w = 1, or all zero for a seed without a ray).  Poses are the
 * caller's: it passes them with every known request and keeps them in its own extra section.
 *   dsm_checkpoint_views_enable  once, after dsm_views_enable (DSM_E_STATE before it and when called twice).  From
 *                       then on every file is version 2 (a views section, even with no slot filled) and every journal
 *                       beside such a base carries, per record, exactly the slots captured since the previous checkpoint.
 *                       Enabling in the middle of an incremental chain makes the next incremental checkpoint a base.
 *                       With dsm_checkpoint_enable (either order: the second call allocates it) the checkpoint gains a
 *                       device and a pinned views image of 16 B per ray for max_views x S rays each (28.8 MB each for
 *                       256 views of 1226x370).  DSM_E_NOMEM with nothing kept.
 * Loading (dsm_map_load, dsm_map_load_journal) on a context that opted in replaces its views by the file's: slots not in
 * the file, and every slot for a version-1 file, become unfilled.  Checked before the device is touched: DSM_E_CAPACITY
 * for a slot >= max_views; DSM_E_INVALID for a ray dsm_views_capture cannot have written (w not 0 or 1, w = 0 with a
 * non-zero byte, a non-finite coordinate).  On a context that did not opt in, a file with a views section is DSM_E_STATE
 * and nothing is loaded; views are untouched by a version-1 file.  dsm_map_peek, dsm_map_peek_journal and
 * dsm_journal_materialize read both versions; materialising a version-2 chain writes the version-2 file of its state. */
int dsm_checkpoint_views_enable(dsm_ctx *ctx);

/* ---- exploration frontiers: clusters of known-free voxels that border unknown space (DESIGN.md §8.10) ----
 * A frontier job reads the state grid of the latest field request, which must be a known one (any enqueue call, waited
 * for or not), in stream order behind it, with that request's origin o and voxel edge v captured at the job's enqueue; a
 * later field request may be enqueued while a job is in flight and does not change what the job reads.  Only the state
 * grid is read, never the map.  Voxel (x, y, z) has the linear index (z * ny + y) * nx + x.
 *
 * Definition (integer throughout, so the result does not depend on the schedule; the centroid rounds once per step).
 *   Frontier voxel: state 2 (free) with at least one of its six face neighbours INSIDE the grid of state 0 (unknown);
 *   neighbours outside the grid do not count, so the box's own faces are no frontier.
 *   Components: the 26-connected components of the frontier voxels, ordered by ascending `first`, the lowest linear
 *   index among their voxels (scipy.ndimage.label with a 3x3x3 structure numbers them in this order).
 *   Clusters: the components of at least min_voxels voxels, in the same order.  Per cluster: n_voxels, first, the
 *   inclusive grid-coordinate bounds lo / hi, n_faces the number of (frontier voxel, unknown face neighbour) pairs,
 *   open the sum over those pairs of the unit step toward the unknown neighbour (the direction to look), and
 *   centroid_k = ((double)sum_k / (double)n_voxels + ((double)o_k + 0.5)) * (double)v in world metres, sum_k the exact
 *   sum of the members' grid coordinates.
 *   Capacities: the table holds the first max_clusters clusters.  The voxel list holds the members of listed clusters
 *   as int32 linear indices, grouped by cluster in table order and ascending within one; a cluster's offset is the
 *   exclusive prefix sum of n_voxels over the table, or -1 when offset + n_voxels > max_voxels, so the list always holds
 *   whole clusters, and they are a prefix of the table.
 *   Counts: n_frontier every frontier voxel, n_components every component, n_clusters every cluster (the table holds
 *   min(n_clusters, max_clusters)), n_listed the voxels in the list.  No free or no unknown voxel: all counts are 0.
 *
 *   dsm_frontier_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID
 *                          for a negative capacity or one above 2^26.  Allocates, for the field's grid and in the worst
 *                          case (at most ceil(nx/2) ceil(ny/2) ceil(nz/2) components), a label grid (4 B per voxel), the
 *                          component and cluster scratch, the device result and its pinned copy of
 *                          32 + 96 max_clusters + 4 max_voxels bytes, and an event.  DSM_E_NOMEM, with nothing kept.
 *   dsm_frontier_enqueue   asynchronous on the context's stream, never waits: the kernels, one D2H copy of the result
 *                          capacity and the event.  DSM_E_STATE before dsm_frontier_enable, before any field request,
 *                          when the latest field request is not a known one, and while a job is in flight;
 *                          DSM_E_INVALID for min_voxels < 1.
 *   dsm_frontier_wait      waits for that job only.  *clusters (min(n_clusters, max_clusters) records) and *voxels
 *                          (n_listed) are the context's pinned results, valid until the next dsm_frontier_enqueue; any
 *                          out-pointer may be NULL.  If the field the job read was taken after a rejected frame, returns
 *                          DSM_E_CAPACITY with valid results and does NOT clear the error, as dsm_field_wait.
 *                          DSM_E_STATE with no job enqueued.
 *   dsm_debug_field_load_state   test entry: makes the caller's state grid (nx * ny * nz bytes, [z][y][x]) at origin
 *                          o the latest known field request, as if a known request had produced it: one H2D copy into
 *                          the grid, the known distance transform and a host copy, waited for with dsm_field_wait and
 *                          read with dsm_field_state like any known request.  DSM_E_INVALID for a byte above 2 or an
 *                          origin outside dsm_field_enqueue's bounds; DSM_E_STATE before dsm_views_enable and while a
 *                          field is in flight. */
typedef struct dsm_frontier_cluster_t
{
    int32_t n_voxels, first, offset; /* offset: into the voxel list, -1 when the cluster is not in it */
    int32_t lo[3], hi[3];            /* inclusive grid-coordinate bounds */
    int32_t reserved;                /* 0 */
    int64_t n_faces, open[3];
    double centroid[3];              /* metres */
} dsm_frontier_cluster_t;            /* 96 B */
typedef struct dsm_frontier_counts_t
{
    int32_t n_frontier, n_components, n_clusters, n_listed;
} dsm_frontier_counts_t;
#define DSM_FRONTIER_MAX_CAPACITY (1 << 26)
int dsm_frontier_enable(dsm_ctx *ctx, int max_clusters, int max_voxels);
int dsm_frontier_enqueue(dsm_ctx *ctx, int min_voxels);
int dsm_frontier_wait(dsm_ctx *ctx, const dsm_frontier_cluster_t **clusters, const int32_t **voxels, dsm_frontier_counts_t *counts);
int dsm_debug_field_load_state(dsm_ctx *ctx, const uint8_t *state, const int32_t origin[3]);

/* ---- the signed distance field: how deep a point lies inside the sites, and a gradient out of them (DESIGN.md §8.16) ----
 * The distance grid is 0 on every site, so a point among sites has dist = 0 and a zero gradient: an optimiser whose path
 * crosses an obstacle or unknown space has no direction to move in.  The signed grid of a request measures that depth.
 *
 * Definition.  S is the request's sites, those its dist measures to: the occupied voxels of a plain (or resident)
 * request, the voxels of state 0 or 1 of a known one (dsm_field_enqueue_known, dsm_debug_field_load_state).  F is every
 * other voxel.  A voxel of F has sdist = dist, bit for bit.  A voxel of S has sdist = (1 - sqrtf((float)e2)) * v in fp32,
 * one rounding per operation, e2 the smallest squared integer distance to a voxel of F (e2 <= 3 * 1023^2, so (float)e2
 * is exact): a site with a face neighbour in F reads 0, as dist does, and the value falls by one voxel edge per voxel of
 * depth, so the slope across the boundary is 1 on both sides.  F empty: -INFINITY everywhere; S empty: +INFINITY
 * everywhere (dist's rule).  So sdist <= dist everywhere, equal off S and on sites with e2 = 1, and sdist < 0 exactly on
 * sites with e2 >= 2.
 *
 * Signed queries.  dsm_field_query_enqueue_signed samples the signed grid with dsm_field_query_enqueue's addressing,
 * interpolation, gradient and clearance, with two rules in place of its "no site" rule: no site gives every inside
 * point +INFINITY and a zero gradient; no voxel of F gives -INFINITY and a zero gradient.  min_dist may be negative (the
 * penetration depth of the path's deepest sample); first_hit is the first inside sample with dist < radius.
 *
 *   dsm_field_signed_enable        once, after dsm_field_enable (DSM_E_STATE before it, when called twice, and while a
 *                                  field is in flight).  Allocates the signed grid (4 B per voxel and 16 B of header) on
 *                                  the device and a pinned host copy of it.  DSM_E_NOMEM with nothing kept.  Every field
 *                                  request enqueued after it, of any kind, also builds the signed grid, in stream order
 *                                  after its distance grid; a request with a host copy also copies the signed grid.
 *   dsm_field_signed               the signed grid [z][y][x] of the last waited request (the context's pinned buffer,
 *                                  valid until the next field enqueue; NULL for a resident request); sdist may be NULL.
 *                                  DSM_E_STATE when that request has no signed grid, or a request has been enqueued since.
 *                                  DSM_E_CAPACITY as dsm_field_wait, with the grid of the last applied frame.
 *   dsm_field_query_enqueue_signed dsm_field_query_enqueue (same arguments, checks, staging and ordering; waited for
 *                                  with dsm_field_query_wait) on the signed grid of the latest field request.  DSM_E_STATE
 *                                  also when that request was enqueued without a signed grid. */
int dsm_field_signed_enable(dsm_ctx *ctx);
int dsm_field_signed(dsm_ctx *ctx, const float **sdist);
int dsm_field_query_enqueue_signed(dsm_ctx *ctx, const double *points, int n_points, const double *waypoints, const int32_t *offsets,
                                   int n_trajectories, float step, float radius);

/* ---- trajectory optimisation on the signed grid: smoothness, clearance and feasibility of B-splines (DESIGN.md §8.17) ----
 * A trajectory job optimises many uniform cubic B-splines, each given by its control points and knot interval, against
 * the signed grid of the latest field request (any kind: plain, resident, known or loaded), in stream order behind it,
 * with that request's origin o and voxel edge v captured at the enqueue.  Like a query it reads only the grid; a later
 * field request may be enqueued while a job is in flight and does not change what the job reads.
 *
 * Definition (every step fp64 with one rounding per operation, except the field samples).
 *   Trajectory j: control points Q_0 .. Q_{N-1} = points[offsets[j] .. offsets[j+1] - 1] (xyz, world metres), 7 <= N <=
 *   256, and knot interval dt = dt[j] > 0.  Q_0..Q_2 and Q_{N-3}..Q_{N-1} are fixed (the start and end state); the free
 *   points are Q_3 .. Q_{N-4}, M = N - 6 of them.
 *   Field term at a free point: d, (gx, gy, gz) the signed point query (dsm_field_query_enqueue_signed) at Q_i in fp32,
 *   widened.  A point outside the grid contributes nothing and is counted; the "no site" rule (+INFINITY) contributes
 *   nothing; a field without a voxel of F (-INFINITY) is not optimised (status 3, the points returned unchanged, every
 *   cost word 0).
 *   Sum: every sum over an index k (a term or a free point, k = i - 3 for free point i) is lane-ordered: lane l = k mod 32
 *   adds its values in ascending k to 0.0, then each lane adds lane l ^ m for m = 16, 8, 4, 2, 1 (the same bits on every
 *   lane).  A product of two per-point vectors sums ((a_x b_x + a_y b_y) + a_z b_z) per point this way.
 *   Cost J = (w_smooth J_s + w_clear J_c) + w_feas J_f:
 *     J_s = sum over m = 0..N-4 of (j_x^2 + j_y^2) + j_z^2, j = (Q_{m+3} - Q_m) + 3 (Q_{m+1} - Q_{m+2}) per axis;
 *     J_c = sum over free points inside the grid with e = margin - d > 0 of e^2;
 *     J_f = F_v + F_a, F_v the sum over m = 0..N-2 of (p_x + p_y) + p_z, p = max(0, V^2 - v_max^2)^2 (zero unless the
 *     difference is > 0) with V = (Q_{m+1} - Q_m) / dt, F_a likewise over m = 0..N-3 with A = ((Q_{m+2} - Q_{m+1}) -
 *     (Q_{m+1} - Q_m)) / dt^2 (dt^2 = dt dt) against a_max^2.
 *   Gradient at free point i, per axis, with D(q) = 4 t q for t = q^2 - lim^2 > 0, else 0:
 *     g_s = 2 (((j_{i-3} - 3 j_{i-2}) + 3 j_{i-1}) - j_i);  g_c = (-2 e) g_axis for a point with a clearance term, else 0;
 *     g_f = (D(V_{i-1}) - D(V_i)) / dt + ((D(A_{i-2}) - 2 D(A_{i-1})) + D(A_i)) / dt^2;
 *     g = (w_smooth g_s + w_clear g_c) + w_feas g_f.
 *   L-BFGS: evaluate at the initial points (evaluations = 1, cost_start = J).  Each iteration: stop with status 0 when
 *   max |g| (from 0.0, fmax) <= g_tol, with status 1 when iterations == max_iter.  Direction: with stored pairs the
 *   two-loop recursion, q = g, for pairs newest to oldest alpha_k = (1 / s_k^T y_k) (s_k^T q), q = q - alpha_k y_k; r =
 *   ((s^T y) / (y^T y) of the newest pair) q; oldest to newest beta = (1 / s_k^T y_k) (y_k^T r), r = r + s_k (alpha_k -
 *   beta); d = -r; if not g^T d < 0 the pairs are dropped.  Without pairs d = -g and the first step is v / sqrt(g^T g),
 *   else 1.  Armijo backtracking: up to max_ls trials x_t = x + step d on the free points, accepted when J_t <= J +
 *   (1e-4 step) g^T d, else step = step 0.5; no accepted trial stops with status 2 at the last accepted point.  After
 *   an accepted trial s = x_t - x, y = g_t - g; the pair is kept (dropping the oldest beyond `memory`) when s^T y > 0.
 *   n_free_outside counts the free points outside the grid at the returned points.
 *   Final check of the returned points: segment m = 0..N-4 at u = (double)s / K, s < K, then the end point (segment
 *   N-4 at u = 1), sample index m K + s; the point ((b0 Q_m + b1 Q_{m+1}) + b2 Q_{m+2}) + b3 Q_{m+3} per axis with
 *   u2 = u u, u3 = u2 u, w = 1 - u, b0 = ((w w) w) / 6, b1 = ((3 u3 - 6 u2) + 4) / 6, b2 = (((3 u2 - 3 u3) + 3 u) + 1) / 6,
 *   b3 = u3 / 6.  Each sample is a signed point query, distance only; min_dist, argmin, first_hit (d < radius) and
 *   n_outside as the trajectory clearance of dsm_field_query_enqueue.  max_v and max_a are the largest per-axis |V| and
 *   |A| of the returned control points, which bound the curve's velocity and acceleration (its convex-hull property).
 *
 *   dsm_trajectory_enable   once, after dsm_field_signed_enable (DSM_E_STATE otherwise).  DSM_E_INVALID for
 *                           max_trajectories or max_points outside [1, 2^24] or max_memory outside [1, 16].  Allocates the
 *                           pinned and device staging, the L-BFGS history (48 max_memory bytes per point), the device
 *                           result and its pinned copy and an event.  DSM_E_NOMEM with nothing kept.
 *   dsm_trajectory_enqueue  stages the request on the calling thread, then enqueues one H2D copy, the kernels, one D2H
 *                           copy of the used result and the event; never waits.  DSM_E_STATE before dsm_trajectory_enable,
 *                           before any field request, when the latest request was enqueued without the signed grid, and
 *                           while a job is in flight.  DSM_E_INVALID for a NULL pointer or params, n_trajectories outside
 *                           [1, max_trajectories], offsets[0] != 0, a trajectory of fewer than 7 or more than 256 points,
 *                           more than max_points points, a non-finite control point or dt, dt <= 0, a weight, margin,
 *                           v_max, a_max or g_tol that is not finite and >= 0, max_iter outside [0, 1024], memory outside
 *                           [1, max_memory], max_ls outside [1, 32], samples outside [1, 64], a radius that is not finite
 *                           and >= 0, more than 2^32 field samples of optimisation (sum of N_j max_iter (max_ls + 1)), or
 *                           more than 2^26 final samples.
 *   dsm_trajectory_wait     waits for that job only.  *records (n_trajectories) and *points (the optimised control points,
 *                           laid out as the request's) are the context's pinned results, valid until the next
 *                           dsm_trajectory_enqueue; any out-pointer may be NULL.  DSM_E_CAPACITY as dsm_field_query_wait
 *                           for a field taken after a rejected frame, with valid results.  DSM_E_STATE with no job
 *                           enqueued. */
typedef struct dsm_trajectory_params_t
{
    double w_smooth, w_clear, w_feas;  /* weights of J_s, J_c and J_f */
    double margin, v_max, a_max;       /* metres, metres per second, metres per second squared */
    double g_tol;                      /* stop when max |g| <= g_tol */
    int32_t max_iter, memory, max_ls;  /* iterations, L-BFGS pairs, Armijo trials */
    int32_t samples;                   /* K: final samples per segment */
    float radius;                      /* first_hit: a final sample with d < radius */
    int32_t reserved[3];               /* 0 */
} dsm_trajectory_params_t;             /* 88 B */
typedef struct dsm_trajectory_t
{
    int32_t status;                    /* 0 converged, 1 max_iter, 2 line search failed, 3 no voxel of F */
    int32_t iterations, evaluations, n_free_outside;
    double cost_start, cost;           /* J at the initial and the returned points */
    double smoothness, clearance, feasibility; /* J_s, J_c, J_f at the returned points, unweighted */
    double max_v, max_a;
    float min_dist;
    int32_t argmin, first_hit, n_outside;
    int32_t reserved[2];               /* 0 */
} dsm_trajectory_t;                    /* 96 B */
typedef struct dsm_trajectory_info_t
{
    int32_t origin[3];                 /* of the field the job read, in voxels */
    int32_t n_trajectories, n_points;
    int32_t n_status[4];               /* trajectories per status */
    int32_t reserved[7];               /* 0 */
} dsm_trajectory_info_t;               /* 64 B */
#define DSM_TRAJECTORY_MAX_POINTS 256
#define DSM_TRAJECTORY_MAX_MEMORY 16
#define DSM_TRAJECTORY_MAX_CAPACITY (1 << 24)
#define DSM_TRAJECTORY_MAX_ITER 1024
#define DSM_TRAJECTORY_MAX_LS 32
#define DSM_TRAJECTORY_MAX_SAMPLES_PER_SEGMENT 64
#define DSM_TRAJECTORY_MAX_WORK (1ull << 32)
#define DSM_TRAJECTORY_MAX_SAMPLES (1 << 26)
int dsm_trajectory_enable(dsm_ctx *ctx, int max_trajectories, int max_points, int max_memory);
int dsm_trajectory_enqueue(dsm_ctx *ctx, const double *points, const int32_t *offsets, const double *dt, int n_trajectories,
                           const dsm_trajectory_params_t *params);
int dsm_trajectory_wait(dsm_ctx *ctx, dsm_trajectory_info_t *info, const dsm_trajectory_t **records, const double **points);

/* ---- paths through known free space: travel cost from a start to every voxel, goals and frontiers (DESIGN.md §8.11) ----
 * A reach job reads the state grid and the distance grid of the latest field request, which must be a known one, in
 * stream order behind it, with that request's origin o and voxel edge v captured at the job's enqueue, and (with
 * with_frontiers) the result of the latest frontier job.  A later field or frontier request may be enqueued while a job
 * is in flight and does not change what the job reads.  The map is never read.  Linear index (z * ny + y) * nx + x.
 *
 * Definition (integer costs, so a converged result does not depend on the schedule, and the round rule below fixes an
 * unconverged one as well).
 *   Traversable: state 2 (free) and dist >= radius, compared in fp32 on the stored distance (metres).  The known
 *   distance measures to the nearest unknown or occupied voxel inside the grid; voxels outside the grid are not seen by
 *   the field, so clearance near the box's faces counts only what is inside.
 *   Moves: the 26-connected moves between traversable voxels, in units of v / 10: face 10, edge 14, corner 17.  In free
 *   space an offset with sorted absolute components a >= b >= c costs chamfer = 10 a + 4 b + 3 c, between 0.98 and 1.12
 *   times its length.  Costs are uint32; UINT32_MAX is "not reached".
 *   Window of voxel g: the Chebyshev box of radius approach (an integer k in [0, 4]) around g, clipped to the grid.
 *   Start: s_k = floor(p_k / (double)v) - o_k of the fp64 start point p.  The job starts from the traversable voxel u
 *   in the window of s minimising (chamfer(u - s), u), which gets cost 0.  start_status 0 such a voxel, 1 s outside the
 *   grid, 2 no traversable voxel in the window; with 1 or 2 nothing is reached.
 *   Cost to go: cost[x] is the least sum of move weights over paths of traversable voxels from u to x (Dijkstra's).
 *   Rounds: the grid is cut into 8x8x8 tiles from voxel (0, 0, 0), edge tiles clipped.  Round 0 schedules u's tile.  In
 *   round r every scheduled tile reads its voxels and its one-voxel halo from buffer r % 2, relaxes to the tile-local
 *   fixed point with the halo frozen and writes its voxels to buffer (r + 1) % 2; a tile that changed a voxel schedules
 *   itself and its 26 neighbour tiles for round r + 1.  The seeded start is round 0's change: u's tile schedules its
 *   neighbours even when no other voxel of it is reached, since u may reach the grid only across the tile's faces.  rounds counts the rounds with a non-empty schedule; the job is
 *   converged when the last of them changed nothing, and stops after max_rounds.  A converged job's costs are
 *   Dijkstra's; an unconverged one's are the latest value of every voxel, each >= the exact cost.
 *   Targets: the goals, then (with_frontiers) the clusters of the latest frontier job's table in table order; the table
 *   holds the first max_targets of them.  For a target voxel g (a goal's voxel, or every member of a cluster) the
 *   viewpoint is the traversable, reached voxel u in the window of g minimising (cost[u] + chamfer(g - u), u); for a
 *   cluster the minimum runs over its members too, ties going to the lowest member.  A record holds cost = cost[u] +
 *   approach, approach = chamfer(g - u), target g, the viewpoint u and the path's offset and length.  status 0 reached,
 *   1 goal outside the grid, 2 nothing reached in the window, 3 a cluster without members in the frontier list (its
 *   offset is -1).  A record of status != 0 has cost UINT32_MAX, approach, viewpoint and path_offset -1 and path_len 0;
 *   its target is the goal's voxel (-1 outside the grid) or the cluster's first voxel.
 *   Paths: from the viewpoint, step to the traversable neighbour p minimising (cost[p] + w(p, x), p) until the start;
 *   on a converged grid that is a tight predecessor.  Every finite cost was written as a neighbour's earlier cost plus a
 *   weight and costs only fall, so the cost falls at every step of an unconverged grid too and the walk ends, with a
 *   weight sum between the exact cost and the reported one.  The list holds the paths start -> viewpoint as linear
 *   indices, in table order; path_offset is the exclusive prefix sum of path_len, or -1 once offset + path_len would pass
 *   max_path_voxels, so the listed paths are a prefix of the reached targets.
 *   Header: the origin; start_voxel u (-1 without one), start_status, start_approach chamfer(u - s) (0 without one);
 *   rounds and converged; n_traversable voxels and n_reached voxels of finite cost; n_goals, n_clusters_total the
 *   frontier table's entries (0 without with_frontiers; those past max_targets are dropped), n_targets the records and
 *   n_path_voxels the listed path voxels.
 *
 *   dsm_reach_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID for
 *                       a capacity that is negative or above 2^26, max_rounds outside [1, 65536], or a grid above 2^27
 *                       voxels (so that 17 (N - 1) plus an approach fits in 32 bits).  Allocates a traversable byte grid,
 *                       two cost grids (4 B per voxel each), the tile stamps and schedules, the device result and its
 *                       pinned copy of 64 + 32 max_targets + 4 max_path_voxels bytes, a pinned cost-grid copy, the goal
 *                       staging and an event.  DSM_E_NOMEM with nothing kept.
 *   dsm_reach_enqueue   asynchronous on the context's stream, never waits: the goals (n_goals x 3 doubles, may be NULL
 *                       for 0) staged into pinned memory and copied with one H2D copy, the kernels (max_rounds round
 *                       launches; a round with an empty schedule exits at once), one D2H copy of the result capacity,
 *                       with host_copy the cost grid as well, and the event.  DSM_E_STATE before dsm_reach_enable, before
 *                       any field request, when the latest field request is not a known one, while a job is in flight,
 *                       and with with_frontiers when the latest frontier job was not enqueued on the latest field
 *                       request (or there is none).  DSM_E_INVALID for a non-finite start or goal, a radius that is not
 *                       finite and >= 0, an approach outside [0, 4], or n_goals outside [0, max_targets].
 *   dsm_reach_wait      waits for that job only.  *targets (n_targets records), *path (n_path_voxels) and *cost (the
 *                       grid [z][y][x], NULL without host_copy) are the context's pinned results, valid until the next
 *                       dsm_reach_enqueue; any out-pointer may be NULL.  If the field the job read was taken after a
 *                       rejected frame, returns DSM_E_CAPACITY with valid results and does NOT clear the error, as
 *                       dsm_field_wait.  DSM_E_STATE with no job enqueued. */
typedef struct dsm_reach_target_t
{
    uint32_t cost;                   /* cost[viewpoint] + approach, units of v / 10; UINT32_MAX unless status 0 */
    int32_t approach, target, viewpoint;
    int32_t path_offset, path_len;   /* into the path list, -1 when the path is not in it */
    int32_t status, reserved;        /* reserved 0 */
} dsm_reach_target_t;                /* 32 B */
typedef struct dsm_reach_info_t
{
    int32_t origin[3];
    int32_t start_voxel, start_status, start_approach;
    int32_t rounds, converged;
    int32_t n_traversable, n_reached;
    int32_t n_goals, n_clusters_total, n_targets, n_path_voxels;
    int32_t reserved[2];
} dsm_reach_info_t;                  /* 64 B */
#define DSM_REACH_MAX_CAPACITY (1 << 26)
#define DSM_REACH_MAX_ROUNDS 65536
#define DSM_REACH_MAX_VOXELS (1 << 27)
#define DSM_REACH_MAX_APPROACH 4
int dsm_reach_enable(dsm_ctx *ctx, int max_targets, int max_path_voxels, int max_rounds);
int dsm_reach_enqueue(dsm_ctx *ctx, const double start[3], float radius, int approach, const double *goals, int n_goals,
                      int with_frontiers, int host_copy);
int dsm_reach_wait(dsm_ctx *ctx, dsm_reach_info_t *info, const dsm_reach_target_t **targets, const int32_t **path,
                   const uint32_t **cost);

/* ---- driving paths on the terrain: the reach job on the latest terrain job's plane (DESIGN.md §8.21) ----
 * A terrain reach job is the reach job above run on the grid of the latest terrain job (§8.20), in stream order behind
 * that job, which may still be in flight; a later terrain, field or frontier request overwrites what it reads only behind
 * it.  It uses the reach job's buffers, records, info and wait.  Everything not restated here is §8.11's, on that grid.
 *   Grid: the terrain grid m (m[|up| - 1] = 1) at the terrain job's origin, voxel edge v.  Cells in the terrain planes'
 *   linear order q P + p, P and Q the two in-plane extents, p and q the lower and higher in-plane axes; start_voxel,
 *   target, viewpoint, the path list and the cost grid are cells.  The header's origin is the terrain job's.
 *   Traversable: status 2 and clearance >= radius, dsm_traversable on the status and clearance planes.
 *   Moves: the 8 in-plane moves, face 10 and diagonal 14, in units of v / 10.  The cost is horizontal travel only: every
 *   traversable cell has step <= max_step, so no move between two of them climbs more than max_step voxels.
 *   Start and goals: a point's voxel as in §8.11 with its up coordinate replaced by 0, so a point's column is where a
 *   ground robot stands whatever its height; status 1 is decided by the two in-plane axes.  The window is a square.
 *   Frontier targets: every member voxel of the latest frontier job stands for its column's cell; ties go to the lowest
 *   member in the field's voxel order; a record's target is the cell of that member, or of the cluster's first voxel
 *   for status 2 and 3.  Members sharing a column are allowed.
 *   Rounds: tiles of 32 x 16 cells from cell (0, 0), 32 along p and 16 along q; a tile that changed schedules itself
 *   and its 8 in-plane neighbours.  The round-0 rule, rounds and converged are §8.11's; a converged job is Dijkstra's on
 *   the 8-connected graph.
 *
 *   dsm_reach_enqueue_terrain  as dsm_reach_enqueue.  DSM_E_STATE before dsm_reach_enable, with no terrain job yet,
 *                              while a reach job is in flight, and with with_frontiers unless the latest frontier job
 *                              read the field request the latest terrain job read.  DSM_E_INVALID exactly as
 *                              dsm_reach_enqueue.  dsm_reach_wait's *cost then holds m0 m1 m2 cells, and it returns
 *                              DSM_E_CAPACITY when the terrain job's field was taken after a rejected frame.  The job
 *                              reads no field request, so a field viewpoint job's with_reach refuses its cost grid; a
 *                              terrain viewpoint job's (§8.23) takes it while the job ran on the latest terrain job. */
int dsm_reach_enqueue_terrain(dsm_ctx *ctx, const double start[3], float radius, int approach, const double *goals, int n_goals,
                              int with_frontiers, int host_copy);

/* ---- travel costs between many sites: the cost matrix of an exploration tour (DESIGN.md §8.13) ----
 * A matrix job reads the state and distance grids of the latest field request, which must be a known one, in stream
 * order behind it, with that request's origin o and voxel edge v captured at the job's enqueue, as a reach job does.
 * It shares no buffer with the reach job.  Everything not restated here is §8.11's: traversable, the moves and their
 * weights, the approach window, the 8x8x8 tiles and the round rule with round 0's seeded start tile.
 *   Sites: site i is the fp64 point points[3i..3i+2], snapped exactly as a reach job snaps its start: voxel u_i,
 *   status_i (0 ok, 1 outside the grid, 2 no traversable voxel in the window) and approach_i = chamfer(u_i - s_i).  A
 *   traversable voxel's centre ((o + x) + 0.5) v snaps to itself.  Points may repeat.
 *   Active tiles: the tiles holding a traversable voxel, numbered in tile order; n_active_tiles of them.  With
 *   n_active_tiles > max_tiles the job has status 1 (capacity): every matrix entry is UINT32_MAX and every site record
 *   holds its snap with rounds = converged = n_reached = 0.  The cut depends on the grid and the radius only.
 *   Costs: for a site of status 0, cost_i is the cost grid of a reach job started at u_i with the same radius, approach
 *   and max_rounds, bit for bit, unconverged values included; its rounds, converged and n_reached are that job's.  A
 *   site of status 1 or 2 reaches nothing, with rounds 0 and converged 1, as such a reach job.
 *   Matrix: M[i][j] = cost_i[u_j] when the job and both sites have status 0, UINT32_MAX otherwise; M[i][i] = 0, and M
 *   is symmetric between converged sites.  The approaches are not added.
 *   Header: the origin, n_sites, status, n_traversable, n_active_tiles, max_tiles and rounds (the launches whose
 *   schedule was non-empty for some site).
 *
 *   dsm_reach_matrix_enable   once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).
 *                             DSM_E_INVALID for max_sites outside [1, 1024], max_tiles outside [1, tiles of the grid],
 *                             max_rounds outside [1, 65536], a grid above 2^27 voxels, or cost buffers (4 KB per site
 *                             and tile) above 2^34 bytes.  DSM_E_NOMEM with nothing kept.
 *   dsm_reach_matrix_enqueue  asynchronous on the context's stream, never waits: the points' voxels staged into pinned
 *                             memory and copied with one H2D copy, the kernels (max_rounds round launches; a round with
 *                             an empty schedule exits at once), one D2H copy of 64 + 32 n + 4 n^2 bytes and the event.
 *                             DSM_E_STATE before dsm_reach_matrix_enable, before any field request, when the latest
 *                             field request is not a known one, and while a job is in flight.  DSM_E_INVALID for a
 *                             non-finite point, a radius that is not finite and >= 0, an approach outside [0, 4],
 *                             n_points outside [1, max_sites], or n_points x max_tiles x max_rounds above 2^32.
 *   dsm_reach_matrix_wait     waits for that job only.  *sites (n_sites records) and *matrix (n_sites x n_sites, row i
 *                             from site i) are the context's pinned results, valid until the next
 *                             dsm_reach_matrix_enqueue; any out-pointer may be NULL.  DSM_E_CAPACITY with valid results
 *                             after a rejected frame, without clearing the error, as dsm_reach_wait.  DSM_E_STATE with
 *                             no job enqueued. */
typedef struct dsm_reach_site_t
{
    int32_t voxel, status, approach;   /* voxel -1 and approach 0 unless status 0 */
    int32_t rounds, converged, n_reached;
    int32_t reserved[2];               /* 0 */
} dsm_reach_site_t;                    /* 32 B */
typedef struct dsm_reach_matrix_info_t
{
    int32_t origin[3];
    int32_t n_sites, status;
    int32_t n_traversable, n_active_tiles, max_tiles, rounds;
    int32_t reserved[7];               /* 0 */
} dsm_reach_matrix_info_t;             /* 64 B */
#define DSM_REACH_MATRIX_MAX_SITES 1024
#define DSM_REACH_MATRIX_MAX_COST_BYTES (1ull << 34)
#define DSM_REACH_MATRIX_MAX_WORK (1ull << 32)
int dsm_reach_matrix_enable(dsm_ctx *ctx, int max_sites, int max_tiles, int max_rounds);
int dsm_reach_matrix_enqueue(dsm_ctx *ctx, const double *points, int n_points, float radius, int approach);
int dsm_reach_matrix_wait(dsm_ctx *ctx, dsm_reach_matrix_info_t *info, const dsm_reach_site_t **sites, const uint32_t **matrix);

/* ---- driving costs between many sites: the matrix job on the latest terrain job's plane (DESIGN.md §8.22) ----
 * A terrain matrix job is the matrix job above run on the plane of the latest terrain job (§8.20), as the terrain reach
 * job (§8.21) runs the reach job there: in stream order behind that job, which may still be in flight; a later terrain,
 * field or frontier request overwrites what it reads only behind it.  It uses the matrix job's buffers, enable, info,
 * site records, result and wait, and allocates nothing.  Everything not restated here is §8.13's, on that plane.
 *   Grid: §8.21's, the plane (P, Q, 1) at the terrain job's origin and voxel edge v, cells in the linear order q P + p;
 *   site voxels are cells, and the header's origin is the terrain job's.
 *   Traversable: status 2 and clearance >= radius, as in §8.21; the 8 in-plane moves, face 10 and diagonal 14.
 *   Sites: a point is snapped as a terrain reach job's start: its column (its up coordinate replaced by 0), then the
 *   approach window as a square; status 1 is decided by the two in-plane axes.  A cell centre, in-plane coordinates
 *   ((o_h + c_h) + 0.5) v and any up coordinate, snaps to itself, so a terrain reach job's viewpoint cells may come back
 *   as sites.
 *   Active tiles: the 32 x 16 tiles from cell (0, 0) that hold a traversable cell, in tile order; status 1 (the cut)
 *   when n_active_tiles > max_tiles.
 *   Costs: for a site of status 0, its row reads the cost plane of a dsm_reach_enqueue_terrain job started there with
 *   the same radius, approach and max_rounds, bit for bit, unconverged values included; its rounds, converged and
 *   n_reached are that job's.  M[i][j] = cost_i[u_j] as in §8.13.
 *
 *   dsm_reach_matrix_enqueue_terrain  as dsm_reach_matrix_enqueue.  DSM_E_STATE before dsm_reach_matrix_enable, with no
 *                                     terrain job yet, and while a matrix job is in flight.  DSM_E_INVALID exactly as
 *                                     dsm_reach_matrix_enqueue, the n_points x max_tiles x max_rounds <= 2^32 bound
 *                                     included.  dsm_reach_matrix_wait returns DSM_E_CAPACITY when the terrain job's
 *                                     field was taken after a rejected frame.  The job reads no field request.  Terrain
 *                                     and field matrix jobs may alternate on one context. */
int dsm_reach_matrix_enqueue_terrain(dsm_ctx *ctx, const double *points, int n_points, float radius, int approach);

/* ---- the order of an exploration tour: multi-start local search over a travel-cost matrix (DESIGN.md §8.14) ----
 * A tour job orders n sites by a deterministic multi-start local search for the asymmetric TSP over a row-major uint32
 * matrix M[i][j] (the cost from i to j, UINT32_MAX: no path), such as the matrix of dsm_reach_matrix_wait as it stands.
 * It reads no field and no map: it has no pairing rule with a field request and no DSM_E_CAPACITY after a rejected
 * frame.  All arithmetic is int64, so the result does not depend on the schedule.
 *   Included sites: site 0 (the robot) and every j >= 1 with M[0][j] != UINT32_MAX, n_included = m of them; the others
 *   are left out of the tour.  A matrix job's sites of status != 0 fall out, their row and column being UINT32_MAX.
 *   Weights: w(i, i) = 0 (the diagonal is ignored), w(i, 0) = 0 when open, else w(i, j) = M[i][j], or P = 2^42 for
 *   UINT32_MAX.  P exceeds any sum of 1024 finite entries, so a tour with fewer unreachable legs always costs less.
 *   Tour: positions 0..m-1, t_0 = 0 and t_m = t_0; cost C = sum over k < m of w(t_k, t_{k+1}) (open: the path from the
 *   robot, the leg back being free; closed: a tour back to site 0); n_infinite counts the legs priced P.
 *   Construction of start s: positions k = 1..m-1 in turn, among the c = min(3, unvisited) unvisited included sites of
 *   least (w(t_{k-1}, j), j): start 0 takes the first (nearest neighbour), start s >= 1 candidate
 *   splitmix64(seed ^ ((uint64)s << 32) ^ k) % c, splitmix64(x) being the splitmix64 generator's output for state x
 *   (x += 0x9e3779b97f4a7c15, then its finaliser).
 *   Passes: up to max_passes, each over the whole neighbourhood: 2-opt reverses positions [i, j], 1 <= i < j <= m-1;
 *   Or-opt moves positions [i, i+L-1], L in {1, 2, 3}, i >= 1, i+L-1 <= m-1, unreversed into the gap after position q,
 *   q in [0, m-1] outside [i-1, i+L-1].  A pass applies the move of least (delta, type (2-opt 0, Or-opt 1), i, L (2-opt
 *   0), j or q) when its delta is negative; otherwise the start has converged.  passes counts the applied moves, so a
 *   start converged exactly when passes < max_passes.
 *   Result: the best start is the least (C, s).  The header, one record per start and the best tour's order (order[0] =
 *   0, -1 past n_included): 64 + 16 n_starts + 4 n bytes.
 *
 *   dsm_tour_enable   once per context (DSM_E_STATE when called twice).  DSM_E_INVALID for max_sites outside [1, 1024]
 *                     or max_starts outside [1, 1024].  Allocates the pinned and device matrix (4 max_sites^2 bytes
 *                     each), the starts' tours (4 max_sites max_starts bytes), the device result and its pinned copy and
 *                     an event.  DSM_E_NOMEM with nothing kept.
 *   dsm_tour_enqueue  asynchronous on the context's stream, never waits: the matrix staged into pinned memory on the
 *                     calling thread, one H2D copy of 4 n^2 bytes, the kernels, one D2H copy of the used result and the
 *                     event.  DSM_E_STATE before dsm_tour_enable and while a job is in flight.  DSM_E_INVALID for a NULL
 *                     matrix, n outside [1, max_sites], n_starts outside [1, max_starts], open not 0 or 1, max_passes
 *                     outside [0, 65536], or n_starts x max_passes x n^2 above 2^32 (this bounds the work of one call).
 *   dsm_tour_wait     waits for that job only.  *starts (n_starts records) and *order (n entries) are the context's
 *                     pinned results, valid until the next dsm_tour_enqueue; any out-pointer may be NULL.  DSM_E_STATE
 *                     with no job enqueued. */
typedef struct dsm_tour_info_t
{
    int32_t n_sites, n_included, open, n_starts, max_passes, best_start;
    int64_t best_cost;
    uint64_t seed;
    int32_t n_infinite;
    int32_t reserved[5];               /* 0 */
} dsm_tour_info_t;                     /* 64 B */
typedef struct dsm_tour_start_t
{
    int64_t cost;
    int32_t passes, converged;
} dsm_tour_start_t;                    /* 16 B */
#define DSM_TOUR_MAX_SITES 1024
#define DSM_TOUR_MAX_STARTS 1024
#define DSM_TOUR_MAX_PASSES 65536
#define DSM_TOUR_MAX_WORK (1ull << 32)
#define DSM_TOUR_P (1ll << 42)
int dsm_tour_enable(dsm_ctx *ctx, int max_sites, int max_starts);
int dsm_tour_enqueue(dsm_ctx *ctx, const uint32_t *matrix, int n, int open, int n_starts, int max_passes, uint64_t seed);
int dsm_tour_wait(dsm_ctx *ctx, dsm_tour_info_t *info, const dsm_tour_start_t **starts, const int32_t **order);

/* ---- view gain: the unknown, frontier and cluster voxels a camera pose would see (DESIGN.md §8.12) ----
 * A gain job reads the state grid of the latest field request, which must be a known one, in stream order behind it,
 * with that request's origin o and voxel edge v (widened to fp64) captured at the job's enqueue, and (with clusters)
 * the result of the latest frontier job.  A later field or frontier request may be enqueued while a job is in flight and
 * does not change what the job reads.  The map is never read.  Linear index (z * ny + y) * nx + x.
 *
 * Definition (every step fp64, one rounding per operation; integer counts, so the result does not depend on the
 * schedule).  The camera is a pinhole in the convention of the frames (x right, y down, z forward); view j has the pose
 * [R | t] poses[12 j ..] (row-major, camera to world) and, with clusters, names clusters[j] (an index into the latest
 * frontier job's table, or -1 for none).  For every grid voxel x:
 *   Centre: c_k = ((double)(o_k + x_k) + 0.5) * v and d = c - t.
 *   Frustum: (d_0^2 + d_1^2) + d_2^2 <= Rm * Rm with Rm = (double)max_range; q_z > 0 where q_m = (R_0m d_0 + R_1m d_1)
 *   + R_2m d_2 (R^T d); u = fx (q_x / q_z) + cx with 0 <= u < width; w = fy (q_y / q_z) + cy with 0 <= w < height.
 *   Seen: a frustum voxel whose walk from a = t to b = c, the Amanatides-Woo walk of dsm_field_enqueue_known literally
 *   (w_a = a / v, e = floor(b / v), the same tM and tD, the lowest axis on ties, the same stop when tM > 1), reaches e,
 *   every voxel it visits before e lying inside the grid and, with unknown_blocks = 1 (pessimistic), being free, or,
 *   with unknown_blocks = 0 (optimistic), not being occupied.  For every voxel x of the grid e is o + x (c / v lies
 *   within a few ulp of o + x + 0.5), so e is x itself.  A camera whose voxel floor(t / v) - o lies outside the grid
 *   sees nothing.
 *   Frontier voxel: that of dsm_frontier_enqueue (free, with a face neighbour of state 0 inside the grid), taken from
 *   the state grid itself, so it does not depend on a frontier job.
 *   Record: n_frustum the frustum voxels; n_free, n_unknown, n_occupied the seen voxels of each state; n_frontier the
 *   seen frontier voxels; n_cluster the seen members (voxels of the frontier list) of the named cluster, -1 when no
 *   cluster is named or it has no members in the list; status 0 ok, 1 the camera's voxel lies outside the grid, then
 *   (only with a camera inside) 3 the named cluster is past the table's entries, 2 it is in the table but not in the
 *   voxel list (offset -1).
 *   Header: the origin, n_views, n_clusters_table the frontier table's entries (min(n_clusters, max_clusters); 0
 *   without clusters) and unknown_blocks.
 *
 *   dsm_gain_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID for
 *                      max_views outside [1, 2^20].  Allocates the pinned and device staging of max_views poses, boxes
 *                      and clusters, a cluster-slot grid (4 B per voxel), the device result and its pinned copy of
 *                      32 + 32 max_views bytes, and an event.  DSM_E_NOMEM with nothing kept.
 *   dsm_gain_enqueue   asynchronous on the context's stream, never waits: per view a box is computed and staged with the
 *                      pose and the cluster on the calling thread (the box only sizes the work: see DESIGN.md §8.12),
 *                      then one H2D copy, the kernels, one D2H copy of 32 + 32 n_views bytes and the event.  clusters
 *                      may be NULL (no view names a cluster).  DSM_E_STATE before dsm_gain_enable, before any field
 *                      request, when the latest field request is not a known one, while a job is in flight, and with
 *                      clusters when the latest frontier job was not enqueued on the latest field request (or there is
 *                      none).  DSM_E_INVALID for fx, fy not finite and > 0, cx, cy not finite, width or height outside
 *                      [1, 65536], max_range not finite and > 0 or above 128 v, unknown_blocks not 0 or 1, a non-finite
 *                      pose entry, a cluster index below -1, n_views outside [0, max_views], or a work bound
 *                      n_views (2 ceil(max_range / v) + 3)^3 above 2^31 voxels (this bounds the work of one call).
 *   dsm_gain_wait      waits for that job only.  *gains (n_views records) are the context's pinned results, valid until
 *                      the next dsm_gain_enqueue; either out-pointer may be NULL.  If the field the job read was taken
 *                      after a rejected frame, returns DSM_E_CAPACITY with valid results and does NOT clear the error, as
 *                      dsm_field_wait.  DSM_E_STATE with no job enqueued. */
typedef struct dsm_gain_camera_t
{
    double fx, fy, cx, cy;
    int32_t width, height;
    float max_range;                 /* metres */
    int32_t unknown_blocks;          /* 1: only free voxels pass a line of sight; 0: every voxel but occupied ones */
} dsm_gain_camera_t;                 /* 48 B */
typedef struct dsm_view_gain_t
{
    int32_t n_frustum, n_free, n_unknown, n_occupied, n_frontier, n_cluster;
    int32_t status, reserved;        /* reserved 0 */
} dsm_view_gain_t;                   /* 32 B */
typedef struct dsm_gain_info_t
{
    int32_t origin[3];
    int32_t n_views, n_clusters_table, unknown_blocks;
    int32_t reserved[2];
} dsm_gain_info_t;                   /* 32 B */
#define DSM_GAIN_MAX_VIEWS (1 << 20)
#define DSM_GAIN_MAX_RANGE_VOXELS 128
#define DSM_GAIN_MAX_WORK (1ll << 31)
int dsm_gain_enable(dsm_ctx *ctx, int max_views);
int dsm_gain_enqueue(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *poses, const int32_t *clusters, int n_views);
int dsm_gain_wait(dsm_ctx *ctx, dsm_gain_info_t *info, const dsm_view_gain_t **gains);

/* ---- viewpoints of frontier clusters: clear candidate positions scored at their best heading (DESIGN.md §8.15) ----
 * A viewpoint job reads the state and distance grids of the latest field request, which must be a known one, in stream
 * order behind it, with that request's origin o and voxel edge v (widened to fp64) captured at the job's enqueue; the
 * result of the latest frontier job, which must have read that request; and with with_reach the cost grid of the latest
 * reach job, which must have read it too.  Later field, frontier and reach requests may be enqueued while a job is in
 * flight and do not change what the job reads.  The map is never read.  Linear index (z * ny + y) * nx + x.
 *
 * Definition (integer counts and gain's fp64 steps, one rounding per operation, so the result does not depend on the
 * schedule).  The camera is dsm_gain_camera_t with gain's meaning; rotation r is rotations[9 r ..], a row-major 3x3
 * camera-to-world matrix.  clusters[i] names an entry of the frontier table.  Per cluster:
 *   Status: 3 the cluster is past the table's entries, 2 it is in the table but not in the voxel list (offset -1), 0
 *   otherwise.  A cluster of status 2 or 3 has no candidates, no samples and no viewpoints.
 *   Centre voxel: g_k = floor(centroid_k / v) - o_k of the table's fp64 centroid (reach's start snap); it lies within
 *   the cluster's lo / hi bounds.
 *   Offsets: every (dx, dy, dz) with all three components multiples of stride, |dz| <= dz_max and r_min^2 <= dx^2 + dy^2
 *   <= r_max^2, enumerated dz outermost, then dy, then dx, each ascending; the offset index is the position in that
 *   list, n_offsets its length.
 *   Candidates: c = g + offset inside the grid and traversable (state free, stored fp32 distance >= radius); with
 *   with_reach also of finite cost in the reach job, that cost being recorded (UINT32_MAX without with_reach).  The
 *   camera sits at the centre t_k = ((double)(o_k + c_k) + 0.5) v.
 *   Samples: with n listed members and n_s = min(n, max_samples), sample k is the member at list position
 *   floor(k n / n_s) (int64); with n <= max_samples every member.
 *   Score: seen[r] counts the samples m whose centre passes gain's frustum test for the pose [R_r | t] and whose walk
 *   from t under unknown_blocks reaches it; n_seen = max_r seen[r], the lowest r on ties.  With every member sampled
 *   seen[r] equals the n_cluster of a gain job on the pose [R_r | t] naming the cluster.
 *   Viewpoints: the candidates with n_seen >= max(1, min_seen), ranked by (-n_seen, cost, offset index); the first top_k.
 *   Records: per cluster the table index, status, n_samples, n_inside (offsets inside the grid), n_traversable, n_reached
 *   (n_traversable without with_reach) and n_viewpoints; then top_k slots per cluster of voxel (linear index), offset
 *   index, rotation, n_seen and cost, an empty slot holding voxel = offset = rotation = -1, n_seen 0 and cost
 *   UINT32_MAX.
 *   Header: the origin, n_clusters, n_offsets, n_rotations, top_k, unknown_blocks, with_reach and n_clusters_table the
 *   frontier table's entries.  The result is 64 + 32 n_clusters (1 + top_k) bytes.
 *
 *   dsm_viewpoint_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).
 *                           DSM_E_INVALID for max_clusters outside [1, 4096] or max_candidates outside [1, 2^22].
 *                           Allocates the pinned and device staging, the per-candidate keys and list, the device result
 *                           and its pinned copy of 64 + 32 max_clusters (1 + 16) bytes, and an event.  DSM_E_NOMEM with
 *                           nothing kept.
 *   dsm_viewpoint_enqueue   asynchronous on the context's stream, never waits: the offsets, rotations and clusters staged
 *                           and copied with one H2D copy, the kernels, one D2H copy of the used result and the event.
 *                           DSM_E_STATE before dsm_viewpoint_enable, before any field request, when the latest field
 *                           request is not a known one, while a job is in flight, when the latest frontier job was not
 *                           enqueued on the latest field request (or there is none), and with with_reach when the latest
 *                           reach job was not either.  DSM_E_INVALID for a NULL camera, params or rotations, NULL
 *                           clusters with n_clusters > 0, gain's camera checks, n_rotations outside [1, 64], a non-finite
 *                           rotation entry, n_clusters outside [0, max_clusters], a cluster index below 0, r_min, r_max
 *                           outside 0 <= r_min <= r_max <= 64, dz_max outside [0, 16], stride outside [1, 8],
 *                           max_samples outside [1, 4096], min_seen < 0, top_k outside [1, 16], with_reach not 0 or 1, a
 *                           radius that is not finite and >= 0, n_offsets outside [1, 4096], n_clusters n_offsets above
 *                           max_candidates, or n_clusters n_offsets max_samples above 2^31 walks (this bounds the work
 *                           of one call).
 *   dsm_viewpoint_wait      waits for that job only.  *clusters (n_clusters records) and *viewpoints (n_clusters x
 *                           top_k slots) are the context's pinned results, valid until the next dsm_viewpoint_enqueue;
 *                           any out-pointer may be NULL.  If the field the job read was taken after a rejected frame,
 *                           returns DSM_E_CAPACITY with valid results and does NOT clear the error, as dsm_field_wait.
 *                           DSM_E_STATE with no job enqueued. */
typedef struct dsm_viewpoint_params_t
{
    int32_t r_min, r_max;            /* horizontal ring, voxels */
    int32_t dz_max, stride;          /* voxels */
    int32_t max_samples, min_seen, top_k, with_reach;
    float radius;                    /* metres: the traversable rule of DESIGN.md §8.11 */
    int32_t reserved;                /* ignored */
} dsm_viewpoint_params_t;            /* 40 B */
typedef struct dsm_viewpoint_cluster_t
{
    int32_t cluster, status, n_samples;
    int32_t n_inside, n_traversable, n_reached, n_viewpoints;
    int32_t reserved;                /* 0 */
} dsm_viewpoint_cluster_t;           /* 32 B */
typedef struct dsm_viewpoint_t
{
    int32_t voxel, offset, rotation, n_seen;   /* voxel -1: an empty slot */
    uint32_t cost;                   /* the reach job's cost at the voxel, UINT32_MAX without with_reach */
    int32_t reserved[3];             /* 0 */
} dsm_viewpoint_t;                   /* 32 B */
typedef struct dsm_viewpoint_info_t
{
    int32_t origin[3];
    int32_t n_clusters, n_offsets, n_rotations, top_k, unknown_blocks, with_reach, n_clusters_table;
    int32_t reserved[6];             /* 0 */
} dsm_viewpoint_info_t;              /* 64 B */
#define DSM_VIEWPOINT_MAX_CLUSTERS 4096
#define DSM_VIEWPOINT_MAX_CANDIDATES (1 << 22)
#define DSM_VIEWPOINT_MAX_OFFSETS 4096
#define DSM_VIEWPOINT_MAX_ROTATIONS 64
#define DSM_VIEWPOINT_MAX_RADIUS 64
#define DSM_VIEWPOINT_MAX_DZ 16
#define DSM_VIEWPOINT_MAX_STRIDE 8
#define DSM_VIEWPOINT_MAX_SAMPLES 4096
#define DSM_VIEWPOINT_MAX_TOP_K 16
#define DSM_VIEWPOINT_MAX_WORK (1ll << 31)
int dsm_viewpoint_enable(dsm_ctx *ctx, int max_clusters, int max_candidates);
int dsm_viewpoint_enqueue(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *rotations, int n_rotations,
                          const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t *params);
int dsm_viewpoint_wait(dsm_ctx *ctx, dsm_viewpoint_info_t *info, const dsm_viewpoint_cluster_t **clusters,
                       const dsm_viewpoint_t **viewpoints);

/* ---- viewpoints of a ground robot: the viewpoint job on the latest terrain job's plane (DESIGN.md §8.23) ----
 * A terrain viewpoint job is the viewpoint job above run on the plane of the latest terrain job (§8.20), as the terrain
 * reach job (§8.21) runs the reach job there: in stream order behind that job, which may still be in flight.  It uses
 * the viewpoint job's buffers, enable, header, records, slots and wait, and allocates nothing.  Its camera stands on the
 * ground: eye voxels above the support of each candidate cell.  Everything not restated here is §8.15's; statuses,
 * samples, scoring, ranking, top_k and the layouts are unchanged.
 *   Plane: §8.21's, the plane (P, Q, 1) at the terrain job's origin o and voxel edge v, cells in the linear order
 *   q P + p, p and q the lower and higher in-plane axes h0 < h1.  A slot's voxel is a cell; the header's origin is the
 *   terrain job's.
 *   Centre cell: reach's start snap of the table's fp64 centroid on the two in-plane axes, floor(centroid_h / v) - o_h:
 *   the centroid's column.
 *   Offsets: §8.15's enumeration with dz_max = 0 (other values are refused); offset (dx, dy) moves along (p, q).
 *   Candidates: c = g + offset inside the plane and traversable, status 2 and clearance >= radius (dsm_traversable on
 *   the status and clearance planes, as §8.21); with with_reach also of finite cost in the latest reach job, which must
 *   be a terrain reach job on the latest terrain job, that cost being recorded.
 *   Camera: at the field voxel whose in-plane coordinates are the cell's (p, q) and whose coordinate along the up axis
 *   a is u = level[c] + eye for a positive up and level[c] - eye for a negative one; t_k = ((double)(o_k + voxel_k) +
 *   0.5) v.  With eye in [1, headroom] of the terrain job, that voxel lies in the grid and is free (the support's
 *   definition), and the camera is (eye - 1/2) v above the support's top face.
 *   Score: §8.15's, with gain's frustum test and walk through the state grid of the field request the terrain job read.
 *   With every member sampled seen[r] equals the n_cluster of a gain job on the pose [R_r | t] naming the cluster.
 *
 *   dsm_viewpoint_enqueue_terrain  as dsm_viewpoint_enqueue.  DSM_E_STATE before dsm_viewpoint_enable, with no terrain
 *                                  job yet, when the latest field request is not the one the latest terrain job read,
 *                                  while a viewpoint job is in flight, when the latest frontier job did not read that
 *                                  request, and with with_reach unless the latest reach job is a terrain reach job on
 *                                  the latest terrain job.  DSM_E_INVALID exactly as dsm_viewpoint_enqueue, and for
 *                                  dz_max != 0 or eye outside [1, headroom].  dsm_viewpoint_wait returns DSM_E_CAPACITY
 *                                  when the terrain job's field was taken after a rejected frame.  Terrain and field
 *                                  viewpoint jobs may alternate on one context. */
int dsm_viewpoint_enqueue_terrain(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *rotations, int n_rotations,
                                  const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t *params, int eye);

/* ---- headings along trajectories: view gain per sample and rotation, then the best rate-limited sequence (DESIGN.md §8.19) ----
 * A heading job reads the state grid of the latest field request, which must be a known one, in stream order behind
 * it, with that request's origin o and voxel edge v (widened to fp64) captured at the job's enqueue.  It needs no
 * frontier job.  A later field request may be enqueued while a job is in flight and does not change what the job reads.
 * The map is never read.
 *
 * Definition (integer counts and int64 scores, so the result does not depend on the schedule; the sample positions fp64
 * with one rounding per operation).
 *   Trajectories: the layout of dsm_trajectory_enqueue, control points Q_0 .. Q_{N-1} = points[offsets[j] ..
 *   offsets[j+1] - 1] of uniform cubic B-splines, 7 <= N <= 256 (dsm_trajectory_wait's optimised points can be passed
 *   unchanged).
 *   Samples: the final-check samples of dsm_trajectory_enqueue at K = samples per segment: segment m = 0..N-4 at u =
 *   (double)s / K, s < K, then the end point (segment N-4 at u = 1); S_j = K (N - 3) + 1 per trajectory, numbered
 *   from sample_offset in trajectory order; the point ((b0 Q_m + b1 Q_{m+1}) + b2 Q_{m+2}) + b3 Q_{m+3} per axis with
 *   that entry's basis, evaluated on the host in that order without contraction.
 *   Rotations: rotations[9 r ..], r < n_rot, row-major 3x3 camera to world as dsm_viewpoint_enqueue takes them.  The list
 *   is a cycle: r and (r +- 1) mod n_rot are neighbouring headings.
 *   Counts: n_unknown[s][r] and n_frontier[s][r] are, by definition, the n_unknown and n_frontier of a gain job with
 *   `camera` on the pose [R_r | p_s]; a sample whose camera voxel floor(p_s / v) - o lies outside the grid counts 0
 *   and adds to n_outside.  score[s][r] = w_unknown n_unknown + w_frontier n_frontier in int64.  Scores add up per
 *   sample: a voxel seen from several samples counts once per sample.
 *   Sequence: r_0 = start; r_{s+1} = (r_s + d_s) mod n_rot with steps d_s in [-max_step, max_step]; with end >= 0,
 *   r_{S-1} = end.  The plan maximises sum_s score[s][r_s], then minimises sum_s |d_s|; remaining ties go to the first
 *   d in the order 0, -1, +1, -2, +2, ... taken sample by sample from s = 0 (distinct d count as distinct even when
 *   they land on the same rotation).  It is a backward pass that keeps the first best successor per (s, r) in that
 *   order, then a forward trace from start.  Status 0 planned; 1 end cannot be reached from start within the limit:
 *   every rotation -1, every turn 0, score and steps 0.
 *   Result: the header; per trajectory its status, n_samples, sample_offset, n_outside, the planned score and steps =
 *   sum |d_s|; per sample its position, rotation and turn, the cumulative signed steps sum_{k<s} d_k from start (for
 *   evenly spaced yaws, yaw_s = yaw_start + turn 2 pi / n_rot, unwrapped); per (sample, rotation) the two counts,
 *   counts[(sample_offset + s) n_rot + r].  The result is 64 + 32 n + 32 S + 8 S n_rot bytes for S samples in all.
 *   Feasibility: the unwrapped yaws, taken as control points of a uniform cubic B-spline with the ends held at knot
 *   interval dt / K (dt the position spline's knot interval), change by at most max_step 2 pi / n_rot between
 *   neighbours, so by the convex-hull property the yaw spline's rate is at most max_step (2 pi / n_rot) K / dt.  That
 *   is why max_step counts list steps per sample interval.  An end that cannot be reached asks for a longer dt or a
 *   free end.
 *
 *   dsm_heading_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID
 *                         for max_trajectories or max_samples outside [1, 2^22].  Allocates the pinned and device
 *                         staging, the device successor table (64 B per sample), the device result and its pinned copy
 *                         of 64 + 32 max_trajectories + 544 max_samples bytes, and an event.  DSM_E_NOMEM with nothing
 *                         kept.
 *   dsm_heading_enqueue   stages the request on the calling thread (the samples and, per sample, a box of grid voxels:
 *                         the hull of gain's boxes over the rotations), then enqueues one H2D copy, the kernels, one D2H
 *                         copy of the used result and the event; never waits.  DSM_E_STATE before dsm_heading_enable,
 *                         before any field request, when the latest field request is not a known one, and while a job
 *                         is in flight.  DSM_E_INVALID for a NULL pointer, n_trajectories outside [1, max_trajectories],
 *                         offsets[0] != 0, a trajectory of fewer than 7 or more than 256 points, a non-finite control
 *                         point, gain's camera checks (with its 128 v range cap), n_rot outside [1, 64], a non-finite
 *                         rotation entry, samples outside [1, 64], a start outside [0, n_rot), an end outside [-1,
 *                         n_rot), a max_step outside [0, n_rot], a weight outside [0, 2^16], more than max_samples
 *                         samples, or more than 2^31 voxel visits, sum_s (2 ceil(max_range / v) + 3)^3 (this bounds the
 *                         work of one call).
 *   dsm_heading_wait      waits for that job only.  *records (n_trajectories), *samples (n_samples) and *counts
 *                         (n_samples x n_rot) are the context's pinned results, valid until the next
 *                         dsm_heading_enqueue; any out-pointer may be NULL.  If the field the job read was taken after a
 *                         rejected frame, returns DSM_E_CAPACITY with valid results and does NOT clear the error, as
 *                         dsm_field_wait.  DSM_E_STATE with no job enqueued. */
typedef struct dsm_heading_request_t
{
    int32_t start;                   /* r_0, in [0, n_rot) */
    int32_t end;                     /* r_{S-1}, in [0, n_rot), or -1: free */
    int32_t max_step;                /* list steps per sample interval, in [0, n_rot] */
    int32_t reserved;                /* ignored */
} dsm_heading_request_t;             /* 16 B */
typedef struct dsm_heading_t
{
    int32_t status;                  /* 0 planned, 1 end unreachable */
    int32_t n_samples, sample_offset, n_outside;
    int64_t score;                   /* sum of the planned rotations' scores */
    int32_t steps;                   /* sum |d_s| */
    int32_t reserved;                /* 0 */
} dsm_heading_t;                     /* 32 B */
typedef struct dsm_heading_sample_t
{
    double p[3];                     /* the sample's position, world metres */
    int32_t rotation;                /* r_s, -1 for status 1 */
    int32_t turn;                    /* sum of the signed steps before s */
} dsm_heading_sample_t;              /* 32 B */
typedef struct dsm_heading_count_t
{
    int32_t n_unknown, n_frontier;
} dsm_heading_count_t;               /* 8 B */
typedef struct dsm_heading_info_t
{
    int32_t origin[3];
    int32_t n_trajectories, n_samples, n_rot, unknown_blocks;
    int32_t n_status[2];             /* trajectories per status */
    int32_t reserved[7];             /* 0 */
} dsm_heading_info_t;                /* 64 B */
#define DSM_HEADING_MAX_CAPACITY (1 << 22)
#define DSM_HEADING_MAX_ROTATIONS 64
#define DSM_HEADING_MAX_SAMPLES_PER_SEGMENT 64
#define DSM_HEADING_MAX_WEIGHT (1 << 16)
#define DSM_HEADING_MAX_WORK (1ll << 31)
int dsm_heading_enable(dsm_ctx *ctx, int max_trajectories, int max_samples);
int dsm_heading_enqueue(dsm_ctx *ctx, const double *points, const int32_t *offsets, int n_trajectories, const dsm_gain_camera_t *camera,
                        const double *rotations, int n_rot, int samples, const dsm_heading_request_t *requests, int32_t w_unknown,
                        int32_t w_frontier);
int dsm_heading_wait(dsm_ctx *ctx, dsm_heading_info_t *info, const dsm_heading_t **records, const dsm_heading_sample_t **samples,
                     const dsm_heading_count_t **counts);

/* ---- terrain: where a ground robot can drive on the known field (DESIGN.md §8.20) ----
 * A terrain job reads the state grid of the latest field request, which must be a known one, in stream order behind it,
 * with that request's origin o captured at the job's enqueue.  A later field request may be enqueued while a job is in
 * flight and does not change what the job reads.  The map is never read.
 *
 * Definition (integer throughout, so the result does not depend on the schedule; the clearance rounds as a field's).
 *   Up axis: up in {+-1, +-2, +-3}, fixed at enable: axis a = |up| - 1 of the field grid, pointing toward +a for a
 *   positive up and -a for a negative one.  "Above voxel k" (k the coordinate along a) is k + 1 for a positive up and
 *   k - 1 for a negative one.  Camera-frame poses with y down (KITTI, the synthetic world) take up = -2; a z-up world
 *   takes up = +3.
 *   Terrain grid: the field grid with axis a collapsed, m_k = n_k except m_a = 1, at the request's origin o (all three
 *   words).  Cell (x, y, z) has the linear index (z * m1 + y) * m0 + x, as a voxel of a grid of shape m.
 *   Support: per column, level = the uppermost (in the up sense) k with state[k] == 1 (occupied) whose `headroom`
 *   voxels above it lie inside the grid and are all of state 2 (free); -1 when no k qualifies.  Unknown space is never
 *   free: a deck whose top no camera has seen is not chosen, and the road under it is when its headroom was observed;
 *   a column whose headroom is cut by the grid's top face or holds one unknown voxel has no support.  The surface of
 *   level k lies at height (o_a + k + 1) v metres along +a for a positive up, and at -(o_a + k) v metres, measured
 *   along -a, for a negative one.
 *   Step: for a cell with support, the largest |level(c) - level(n)| over the cell's in-grid 8-neighbours n in the two
 *   axes other than a that have support, 0 without such a neighbour; 0 for a cell without support.  The result stores
 *   min(step, 255); the status compares the full step.
 *   Status: 0 no support, 1 support but step > max_step, 2 traversable: the field's state codes (unknown, occupied,
 *   free), so "not traversable" is "status != 2".
 *   Clearance: sqrtf((float)d2) * v, d2 the smallest squared integer distance in cells (over the terrain grid) to a cell
 *   of status != 2; 0 on such cells, +inf when every cell is traversable.  It is the known field's distance of the
 *   status plane as a grid of shape m: a caller that keeps clearance >= r keeps a disc of radius r on drivable ground.
 *   Counts: n_support the cells with support, n_blocked those of status 1, n_traversable those of status 2.
 *   Result: per cell an int16 level, a uint8 status, a uint8 step and a float clearance, 8 B per cell.
 *
 *   dsm_terrain_enable    once, after dsm_views_enable (DSM_E_STATE otherwise, and when called twice).  DSM_E_INVALID
 *                         for up outside {+-1, +-2, +-3}.  Allocates, for the field's grid collapsed along a, the device
 *                         result (the four planes, 8 B per cell, and 32 B of header) and its pinned copy, and an event.
 *                         DSM_E_NOMEM with nothing kept.
 *   dsm_terrain_enqueue   asynchronous on the context's stream, never waits: the kernels, one D2H copy of the result and
 *                         the event.  DSM_E_STATE before dsm_terrain_enable, before any field request, when the latest
 *                         field request is not a known one, and while a job is in flight.  DSM_E_INVALID for headroom
 *                         outside [1, n_a - 1] or max_step outside [0, 1023].
 *   dsm_terrain_wait      waits for that job only.  *level, *status, *step and *clearance (m0 m1 m2 cells each) are
 *                         the context's pinned results, valid until the next dsm_terrain_enqueue; any out-pointer may be
 *                         NULL.  If the field the job read was taken after a rejected frame, returns DSM_E_CAPACITY with
 *                         valid results and does NOT clear the error, as dsm_field_wait.  DSM_E_STATE with no job
 *                         enqueued. */
typedef struct dsm_terrain_info_t
{
    int32_t origin[3];               /* the field request's origin, voxels */
    int32_t m[3];                    /* the terrain grid: the field grid with m[|up| - 1] = 1 */
    int32_t up, headroom, max_step;
    int32_t n_support, n_blocked, n_traversable;
    int32_t reserved[4];             /* 0 */
} dsm_terrain_info_t;                /* 64 B */
#define DSM_TERRAIN_MAX_STEP 1023
int dsm_terrain_enable(dsm_ctx *ctx, int up);
int dsm_terrain_enqueue(dsm_ctx *ctx, int headroom, int max_step);
int dsm_terrain_wait(dsm_ctx *ctx, dsm_terrain_info_t *info, const int16_t **level, const uint8_t **status, const uint8_t **step,
                     const float **clearance);

/* ---- checkpoints that do not stop the stream (DESIGN.md §8.5) ----
 * The file of dsm_map_save, taken in stream order like a publish snapshot: the resident stream pays one device-to-device
 * copy of the live map, the transfer to the host runs on a low-priority stream beside the next frames, and a thread of
 * the context writes the file.  For a node that wants a checkpoint every N keyframes without stalling.
 *   dsm_checkpoint_enable   once, on a context with a resident pool (DSM_E_STATE otherwise, and when called twice).
 *                           Allocates a device image and a pinned, mapped host image of
 *                           128 + 44 * max_local_surfels + 56 * (store reservation) bytes each (every section rounded up
 *                           to 128 bytes; 327 MB each at 2 Mi pool + 4 Mi store), a low-priority stream, two events and
 *                           the writer thread, which dsm_destroy joins.  DSM_E_NOMEM.  A later dsm_inactive_reserve
 *                           rebuilds the images at the new size (DSM_E_NOMEM if it cannot; the checkpoint calls then
 *                           return DSM_E_STATE until a reserve succeeds).
 *   dsm_checkpoint_enqueue  asynchronous, ordered on the context's stream exactly like dsm_publish_enqueue.  Copies path
 *                           and extra, captures the geometry and the constants, enqueues the snapshot and the drain and
 *                           hands the write to the thread.  Never waits and reads nothing back.  The file is byte for
 *                           byte what dsm_map_save(ctx, path, extra, extra_bytes) would have written at this position in
 *                           the stream.  DSM_E_INVALID for a NULL path, or extra_bytes > 0 with a NULL extra;
 *                           DSM_E_STATE before dsm_checkpoint_enable, while an earlier checkpoint has not been
 *                           retired by dsm_checkpoint_wait, and, as dsm_map_save, when the context holds no resident
 *                           pool (a batch call since the last dsm_pool_upload) or a dsm_fuse_batch_async batch is in
 *                           flight; nothing is enqueued then and nothing under path changes.  Every other call may run meanwhile (fuses, transforms,
 *                           dsm_map_load, dsm_inactive_load, publishing), except dsm_inactive_reserve (DSM_E_STATE).
 *   dsm_checkpoint_wait     block = 0: DSM_OK with *finished = 0 while the write runs.  Once it has finished (block != 0:
 *                           after waiting for it), returns its result with *finished = 1 and retires the checkpoint:
 *                           DSM_OK once the file is on the disk (temporary name, checksum, fsync, rename, directory
 *                           fsync, as dsm_map_save); DSM_E_IO with nothing left under path; DSM_E_CAPACITY, with no
 *                           file, when a frame of dsm_fuse_stream_window had been rejected before the snapshot -- the
 *                           error is NOT cleared: the next synchronising call reports and clears it, as after
 *                           dsm_publish_wait.  finished may be NULL.  DSM_E_STATE with nothing enqueued.
 * dsm_destroy with a pending checkpoint returns after its file has been written.  A context is still used from one
 * thread at a time; the writer thread touches only the host image and the copies of path and extra.
 *   dsm_debug_checkpoint_drain_ctas   the CTA count of the drain kernel (default 8); DSM_E_STATE while one is pending. */
int dsm_checkpoint_enable(dsm_ctx *ctx);
int dsm_checkpoint_enqueue(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes);
int dsm_checkpoint_wait(dsm_ctx *ctx, int block, int *finished);
int dsm_debug_checkpoint_drain_ctas(dsm_ctx *ctx, int ctas);

/* ---- incremental checkpoints: a journal of changed chunks beside the last full file (DESIGN.md §8.6) ----
 * <path> stays an ordinary dsm_map_save file, the base; <path>.journal holds records, each with the 256-surfel chunks of
 * the pool and the store that changed since the previous checkpoint, the whole segment table and the caller's extra bytes.
 * The chunks are found on the device, by comparing the live map with the checkpoint image of the previous checkpoint, and
 * only changed chunks cross PCIe and reach the disk.
 *   dsm_checkpoint_enqueue_incremental  the contract, ordering and errors of dsm_checkpoint_enqueue; dsm_checkpoint_wait
 *                           retires it.  Writes a base (the file, then a fresh journal header, each under a temporary
 *                           name, flushed and renamed) when it is the first incremental checkpoint to path on this
 *                           context or the previous one went to another path; when the previous checkpoint did not write
 *                           its file or record (DSM_E_CAPACITY, DSM_E_IO); after a dsm_checkpoint_enqueue; after
 *                           dsm_map_load, dsm_map_load_journal, dsm_inactive_load, dsm_inactive_reserve or
 *                           dsm_set_constants; and once the journal has grown larger than its base.  Otherwise appends one
 *                           record and flushes it to the disk.  Either way the state resolved from path afterwards is byte
 *                           for byte what dsm_map_save would have written at this position in the stream.
 *   dsm_map_load_journal    dsm_map_load of the resolved state: the base, then the journal's records in order up to the
 *   dsm_map_peek_journal    first that is torn, fails its checksum, breaks the chain of checksums or is out of sequence.
 *                           A missing journal, or one that names another base, adds nothing.  DSM_E_INVALID for a journal
 *                           of another magic or format, and for a complete record whose chunk lists are not ascending, reach
 *                           past its sizes or miss a chunk that grows a section.  *records (optional): the records applied.
 *                           Otherwise the errors of dsm_map_load / dsm_map_peek on that state.
 *   dsm_journal_materialize writes the file of the resolved state, in its base's version, to out_path (temporary name, fsync, rename),
 *                           without a context: what dsm_map_load reads, for archives and export. */
int dsm_checkpoint_enqueue_incremental(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes);
int dsm_map_load_journal(dsm_ctx *ctx, const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int *records);
int dsm_map_peek_journal(const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt, int seg_cap,
                         int *n_segments, int *records);
int dsm_journal_materialize(const char *path, const char *out_path);

/* ---- multi-GPU: frames of a batch sharded across GPUs, ONE gather of the surfel deltas at the end (SURVEY.md 8e) ----
 * One context per GPU (one process or thread each).  The reference has no counterpart (fuse_initialize_map is
 * single-process, fusion_functions.cpp:30-83); what is gathered is what SurfelMap::fuse_map consumes after the call
 * (surfel_map.cpp:1077-1109): every frame's new surfels and updated local surfels.
 *   dsm_comm_unique_id   rank 0 creates the 128-byte NCCL id and hands it to the other ranks out of band
 *   dsm_comm_init        collective: joins the communicator (ncclCommInitRank); NCCL is dlopen'ed ("libnccl.so.2": inside a
 *                        PyTorch process the copy torch already loaded), DSM_E_NCCL if it is missing
 *   dsm_gather_deltas    collective, after dsm_batch_run: packs ONLY the valid records of this rank's batch
 *                          int32 'DSMD', n_frames, n_new_total, n_pool_total, n_new[n_frames], pool_ofs[n_frames+1], pad to 16 B,
 *                          dsm_surfel_t new[n_new_total] (frame by frame, seed-index order), dsm_surfel_t pool[n_pool_total]
 *                        and moves it to `root` on a side stream.  Ranks of one node write their payload straight into
 *                        their slot of the root's receive buffer over NVLink peer memory (CUDA IPC mapping made at the first
 *                        gather; counts stay on the device, nothing waits on the host, exactly the valid bytes travel);
 *                        without a peer mapping (or with DSM_GATHER_NCCL=1) the counts go to the host and the payloads move
 *                        with ncclAllGather (sizes) + one grouped ncclSend/ncclRecv.  Collective: every rank of the
 *                        communicator calls it with the same root, in the same order.  Returns before the transfer has
 *                        finished; the next dsm_batch_run may be enqueued at once.  A new gather overwrites the previous one.
 *   dsm_gather_wait      root: waits until every rank's payload has arrived; other ranks: until their own has left
 *   dsm_gathered_*       root only: the payload of every rank, on the device (zero copy; payload r occupies
 *                        [rank_offsets[r], rank_offsets[r] + dsm_gathered_rank_bytes(r))) or copied to host memory */
#define DSM_COMM_ID_BYTES 128
int dsm_comm_unique_id(void *id_out128);
int dsm_comm_init(dsm_ctx *ctx, const void *id128, int rank, int nranks);
int dsm_comm_destroy(dsm_ctx *ctx);
int dsm_gather_deltas(dsm_ctx *ctx, int root);
int dsm_gather_wait(dsm_ctx *ctx);
int dsm_gathered_device(dsm_ctx *ctx, void **dev_ptr, size_t *rank_offsets /* [nranks + 1] */);
int dsm_gathered_rank_bytes(dsm_ctx *ctx, int rank, size_t *bytes);
int dsm_gathered_download(dsm_ctx *ctx, int rank, void *host_out, size_t cap);

/* ---- parity / debug readback (what the reference keeps private: fusion_functions.h:34-37) ---- */
int dsm_get_labels(dsm_ctx *ctx, int frame, int32_t *labels_hw);   /* superpixel_index, [H][W] */
int dsm_get_seeds(dsm_ctx *ctx, int frame, dsm_seed_t *seeds_s);   /* superpixel_seeds, [S] */

/* debug: enqueue only the first n kernels of the schedule on the next dsm_batch_run (n <= 0: all).
 * Lets the parity tests localise a mismatch to one pass; never used on the product path. */
int dsm_debug_stop_after(dsm_ctx *ctx, int n_kernels);
/* debug: number of "cannot happen" events the kernels counted in the last batch (a non-stable seed
 * without members, SURVEY.md §7 H3); the parity tests assert it is 0. */
int dsm_debug_invariant_violations(dsm_ctx *ctx, int *count);

/* ---- measurement hooks ----
 * Per-kernel CUDA-event timing on the context's stream.  mask selects kernels (bit k = kernel
 * id k, see dsm_kernel_name); 0 disables.  Accumulates until dsm_profile_reset(). */
#define DSM_NUM_KERNELS 10
int dsm_profile_enable(dsm_ctx *ctx, uint32_t kernel_mask);
int dsm_profile_reset(dsm_ctx *ctx);
/* resolves pending events (synchronises); ms_total/launches are [DSM_NUM_KERNELS] */
int dsm_profile_read(dsm_ctx *ctx, float *ms_total, int32_t *launches);
const char *dsm_kernel_name(int kernel_id);
/* raw device pointers for zero-copy interop (e.g. the multi-GPU gather); which: see DSM_BUF_* */
#define DSM_BUF_NEW_SURFELS 0 /* dsm_surfel_t [max_batch][S] */
#define DSM_BUF_NEW_COUNTS 1  /* int32 [max_batch] */
#define DSM_BUF_LOCAL 2       /* dsm_surfel_t [max_local_surfels] */
int dsm_device_buffer(dsm_ctx *ctx, int which, void **dev_ptr, size_t *bytes);

#ifdef __cplusplus
}
#endif
#endif /* DSM_H */
