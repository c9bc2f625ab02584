// Device-side data layout shared by the kernels (dsm_kernels.cu) and the host driver (dsm_capi.cu).
//
// HBM layout per context (B = max_batch frames, P = H*Wp pitched pixels, S = seeds per frame):
//   gray    u8  [B][H][Wp]      Wp = W rounded up to 16 so every row starts 16-byte aligned
//   depth   f32 [B][H][Wp]      (vector loads, TMA boxes; SURVEY.md section 7 H8)
//   invd    f32 [B][H][Wp]      (float)(1.0 / (double)depth) for depth > 0.01, else 0 (:404-405): what the assign passes read
//   code    u8  [B][H][Wp]      superpixel_index of the reference (fusion_functions.h:37) as the index of the winning
//                               candidate among the pixel's 2x2 candidate seeds (dsm_code_seed): the only label state of
//                               the schedule (1 B/px; the window gathers test it with a byte compare against a position-only pattern)
//   labels  i32 [B][H][Wp]      download buffer: filled from the code plane by dsm_get_labels only
//   seed    float4 [B][S]       (x, y, mean_intensity, mean_depth)  -- the clustering state
//   seed_hl float2 [B][S]       1.0 / (double)mean_depth as hi + lo floats (fp32 cost filter of the assign pass)
//   inv_md  f64 [B][S]          1.0 / (double)mean_depth (exact path of the assign pass, :380)
//   tstable i32 [B][S]          stable flag + raster time stamp: INT_MAX = stable,
//                               -1 = unstable, k >= 0 = un-stabled when raster scan reached k
//   und     i32 [B][S]          depth-list lengths of the queued hard Newton seeds (k_gather -> k_newton_hard)
//   dlist   f32 [B][S][232]     member depths in raster order of the queued hard Newton seeds, one contiguous list per
//                               seed (the lists of the other seeds never leave k_gather's shared memory)
//   hardq   i32 [B][S], nhard i32 [B]   queue of the hard Newton seeds (reset by k_assign2, appended by k_gather)
//   done    i32 [B]             frame-completion tickets of the assign pass
//   errflag i32 [B]             invariant violations (must stay 0)
//   kx, ky  f32 [Wp+16], [H+16] back-projection factors, computed once per context
//   qlist   f32 [B][S][3][232]  centred plane-fit inlier points (k_plane_gather -> k_gn_solve fallback passes)
//   hrec    f64 [B][24][S]      first Gauss-Newton pass sums of the plane fit, field-major
//   pfsum   float4 [B][S][2]    per-seed plane-fit summary
//   plane   float4 [B][S][3]    (n.xyz, view_cos) (posi.xyz, mean_depth) (size, I, x, y)
//   fused   i32 [B][S]          Superpixel_seed::fused
//   list    int2 [B][P]         deferred pixels of the stable relaxation: (pitched raster index, winner)
//   nlist   i32 [B]
//   pool    dsm_surfel_t [max_local]   AoS, ABI layout (44 B) so upload/download are plain copies
//   poolofs i32 [B+1]
//   newsurf dsm_surfel_t [B][S], nnew i32 [B]
//   pose/ipose f32 [B][16] column-major, refidx i32 [B]
#pragma once
#include <cstdint>
#include <cuda.h> // CUtensorMap (types only; the encoder is resolved through the runtime, no libcuda link dependency)
#include <cuda_runtime.h>
#include "../../include/dsm.h"

#define DSM_SP 8
#define DSM_STABLE 0x7fffffff

struct DsmDev
{
    // geometry
    int W, H, Wp, spw, sph, S, B;
    int frame0; // first frame slot this launch works on (chunked copy/compute overlap)
    int Sp; // S rounded up to 32: row stride of the [k][seed] scratch lists
    float fx, fy, cx, cy, fuse_far, fuse_near, camera_f;
    // algorithm constants (dsm_set_constants; fusion_functions.h:12-21).  huber_hi = smallest float >= huber: for every float x,
    // (double)x < huber  <=>  x < huber_hi  and  (double)x >= huber  <=>  x >= huber_hi (the float-vs-double-literal compares)
    double huber, baseline, disparity_error, min_tolerate_diff;
    float huber_hi;
    // per-frame strides in elements
    size_t px_stride; // H*Wp
    // buffers
    const uint8_t *gray;
    const float *depth;
    int32_t *labels;
    float4 *seed;
    double *inv_md;
    int32_t *tstable;
    int32_t *und;       // number of member depths > 0.1 (written for the queued hard Newton seeds only)
    float *dlist;       // [B][S][232] member depths in raster order, one contiguous list per queued hard Newton seed
    int32_t *errflag;   // [B] count of "impossible" events (non-stable seed without members, SURVEY H3)
    float4 *plane;
    const float *kx;    // [Wp+16]: ((float)u - cx) / fx, the per-column factor of back_project (:94)
    const float *ky;    // [H+16]:  ((float)v - cy) / fy
    float *qlist;       // [B][S][3][232] centred plane-fit inlier points
    float4 *pfsum;      // [B][S][2]: (sum n.xyz, max_dist) (mean.xyz, inlier count or 0 if rejected)
    int32_t *fused;
    int2 *list;
    int32_t *nlist;
    dsm_surfel_t *pool;
    const int32_t *poolofs;
    dsm_surfel_t *newsurf;
    int32_t *nnew;
    const float *pose;
    const float *ipose;
    const int32_t *refidx;
    int max_pool_per_frame; // largest per-frame pool slice in this batch (grid sizing)
    // resident views only (nullptr in batch views): the sticky error word of dsm_fuse_stream_window.  While it is set,
    // the fuse / initialise / post-step kernels exit at once, so no frame after a rejected one touches the pool.
    const int32_t *gate;
    // tile path (dsm_tile.cu)
    uint8_t *code;      // [B][H][Wp] label of every pixel as the index (0..3) of the winning candidate among its 2x2 candidate seeds, or DSM_CODE_NONE
    float *invd;        // [B][H][Wp] (float)(1.0 / (double)depth) for depth > 0.01, else 0 (:404-405), written by the first assign pass
    float2 *seed_hl;    // [B][S] 1.0 / (double)mean_depth split into two floats (hi, lo) for the filtered assign pass
    int32_t *hardq;     // [B][S] seeds whose Huber-Newton needs the entry-by-entry classification (k_gather -> k_newton_hard)
    int32_t *nhard;     // [B] queue lengths (reset by k_assign2)
    int32_t *done;      // [B] frame-completion tickets of the assign pass (the last CTA of a frame runs the stable relaxation)
    double *hrec;       // [B][24][S] plane fit, first residual pass: H = sum 2 q q^T (9), the same over out-of-range points (10), their clamped gradient (4), packed (margin, qmax2)
};

// Label code of a pixel: which of its (at most) 2x2 candidate seeds it is labelled with, c = 2*ix + iy over the seed
// columns {xa, xa+1} and rows {ya, ya+1}, xa = floor((x - 4) / 8), ya = floor((y - 4) / 8) (the candidate set depends on
// the pixel position only, :413-422), or DSM_CODE_NONE for a pixel the reference would have left without any label
// (input domain, DESIGN.md 1.3), which is labelled 0.
#define DSM_CODE_NONE 4
__device__ __forceinline__ int dsm_code_seed(int c, int x, int y, int spw)
{
    return c == DSM_CODE_NONE ? 0 : (((y - 4) >> 3) + (c & 1)) * spw + ((x - 4) >> 3) + (c >> 1);
}

// TMA descriptors (cuTensorMapEncodeTiled) of the three per-pixel arrays as [B][H][Wp] tensors; box = one seed tile plus halo
struct DsmMaps
{
    CUtensorMap cod, dep, gry; // label codes (u8), depth (f32), gray (u8)
};
// seed tile of the tile kernels: 8 x 4 superpixels = 64 x 32 pixels, plus a 4-pixel halo (the 16 x 16 windows of
// update_seeds_kernel :481-489 and calculate_sp_depth_norms_kernel :806-811 overlap their neighbours by 8)
#define DSM_TILE_SX 8
#define DSM_TILE_SY 4
#define DSM_TILE_W 76  // box width in elements: 72 used; row pitch 76 words = 12 mod 32, so a quarter-warp reading 16 bytes per lane from 8 consecutive rows hits 32 distinct banks
#define DSM_TILE_H 41  // box height: 40 rows + the down neighbour of the last row (pixel normals)
// gray (u8) box: TMA needs the box start 16-byte aligned in global memory, which 64 bx - 4 is for the 4-byte arrays but
// not for bytes, so the gray box starts DSM_TILE_GX = 12 pixels further left (64 bx - 16) and is 112 bytes wide
#define DSM_TILE_GW 112
#define DSM_TILE_GX 12

enum DsmKernelId
{
    DSM_K_SEED_INIT = 0,
    DSM_K_ASSIGN_FIRST = 1,
    DSM_K_ASSIGN = 2,
    DSM_K_GATHER = 3,       // window gather of update_seeds_kernel + the Huber-Newton passes inside the Huber range
    DSM_K_NEWTON = 4,       // Huber-Newton of the seeds with out-of-range entries (k_newton_hard)
    DSM_K_PLANE_GATHER = 5, // pixel normals + plane-fit gather
    DSM_K_PLANE_SOLVE = 6,  // plane-fit solver
    DSM_K_FUSE = 7,
    DSM_K_INIT_SURFELS = 8,
    DSM_K_REPACK = 9,
};

// launchers (dsm_kernels.cu); nb = frames in this batch
void dsm_launch_repack(const DsmDev &d, int nb, const uint8_t *gray_packed, const float *depth_packed, cudaStream_t s);
void dsm_launch_seed_init(const DsmDev &d, int nb, cudaStream_t s);
void dsm_launch_fuse(const DsmDev &d, int nb, cudaStream_t s);
void dsm_launch_init_surfels(const DsmDev &d, int nb, cudaStream_t s);
void dsm_launch_seeds_export(const DsmDev &d, int frame, dsm_seed_t *out_dev, int raw_md, cudaStream_t s);
void dsm_launch_labels_export(const DsmDev &d, int frame, cudaStream_t s);
// Ordered selection over the pool range of frame slot `frame` (mode / key: pool_pred of dsm_kernels.cu; mode 1 flags the
// selected surfels dead): k_pool_count and k_pool_scan leave the per-block offsets in blkofs and the total in *nsel, then
// k_pool_scatter writes the selected records in pool order to dst.  dst == nullptr: count and scan only.
// DSM_SEL_SCATTER_ONLY: the scatter alone, on the blkofs of a count over the same, unchanged range.  DSM_SEL_PDL:
// PDL-linked launches (a chain whose kernels all begin with pdl_enter).  `upper` >= the range's length sizes the grids.
// Records: int32 pool index, the whole 44-byte surfel, PointXYZI float4 {px, py, pz, color}.
enum DsmRec { DSM_REC_INDEX, DSM_REC_SURFEL, DSM_REC_POINT };
enum { DSM_SEL_PDL = 1, DSM_SEL_SCATTER_ONLY = 2 };
void dsm_launch_pool_select(const DsmDev &d, int frame, int upper, int mode, int key, DsmRec rec, void *dst, int *blkcnt,
                            int *blkofs, int *nsel, cudaStream_t s, int flags = 0);
// fuse_map post-step, in place: holes [capacity], src [capacity], sync [dsm_recycle_sync_len(capacity)] (zeroed once)
void dsm_launch_pool_recycle(const DsmDev &d, int frame, int upper, int *blkcnt, int *blkofs, int *nsel, int32_t *holes, int32_t *src,
                             int32_t *sync, int32_t *ofs_out, cudaStream_t s);
#define DSM_RECYCLE_SEG 1024 // tail slots per segment of k_pool_recycle (one CTA works on a segment at a time)
inline size_t dsm_recycle_sync_len(int capacity) { return 2 + (size_t)capacity / DSM_RECYCLE_SEG + 1; } // {ticket, done, segment flags}
void dsm_launch_pool_transform(const DsmDev &d, int frame, int upper, const float *Wm_dev, cudaStream_t s);
void dsm_launch_set2(int32_t *p, int a, int b, cudaStream_t s);
// camera -> world of dsm_frame_raw_cloud: R row-major (R[3r + c] = R(r, c)) and T, formed on the host
struct DsmRawPose
{
    float R[9], T[3];
};
void dsm_launch_raw_cloud(const DsmDev &d, int frame, const DsmRawPose &pose, float4 *out, cudaStream_t s);
// debug_show of dsm_frame_superpixel_image: out = [H][3*Wp] bytes (16-byte aligned), pixels >= W written as 0
void dsm_launch_superpixel_image(const DsmDev &d, int frame, uint8_t *out, cudaStream_t s);
// tile path (dsm_tile.cu)
int dsm_tile_setup(); // raises the dynamic shared-memory limits of the tile kernels (once per process and device)
void dsm_launch_assign2(const DsmDev &d, int nb, bool first, cudaStream_t s);
void dsm_launch_gather(const DsmDev &d, const DsmMaps &m, int nb, cudaStream_t s);
void dsm_launch_newton2(const DsmDev &d, int nb, cudaStream_t s);
void dsm_launch_plane_gather(const DsmDev &d, const DsmMaps &m, int nb, cudaStream_t s);
void dsm_launch_gn_solve(const DsmDev &d, int nb, cudaStream_t s);

// Window step of dsm_fuse_stream_window (move_add_surfels on the device) and the device side of the inactive store.
// tab: the call's staged lists, [0, B] retire offsets and [B+1, 2B+1] reactivation offsets (relative to the key
// arrays), [2B+2] the call's tag, [2B+3] index of the first reactivation key, retire keys from 2B+4.
#define DSM_WIN_KEYS(B) (2 * (B) + 4)
#define DSM_WIN_CHUNK 1024 // store surfels per CTA step of the compaction
struct DsmWin
{
    const int32_t *tab;
    int t, B;             // frame of the call, table stride
    dsm_surfel_t *store;  // inactive store
    int4 *seg;            // segment table: (keyframe, offset, count, scratch) in retirement order
    int32_t *hdr;         // {store size, segments, surfels the frame reactivates, lowest offset they leave}
    int32_t *res;         // resident offsets {0, pool size, error tag, rejected frame}
    int32_t *blk;         // [DSM_WINDOW_MAX_KEYS][blk_stride] per-key block counts, then store offsets
    int32_t *sync;        // compaction: {ticket, unused, per-chunk "read" flags}, zero between steps
    int blk_stride, pool_cap, store_cap, S;
};
inline size_t dsm_win_sync_len(int store_cap) { return 2 + (size_t)store_cap / DSM_WIN_CHUNK + 2; }
// nr / na: lengths of the frame's retire / reactivation lists (which kernels are needed); `upper` bounds the pool size
void dsm_launch_window_step(const DsmDev &d, const DsmWin &w, int upper, int nr, int na, cudaStream_t s);
// warp_inactive_surfels_cpu_kernel for the segments of keyframe kf, located on the device (w.seg / w.hdr)
void dsm_launch_inactive_transform(const DsmWin &w, int kf, const float *Wm_dev, cudaStream_t s);

// Snapshot header of dsm_publish_enqueue, in pinned host memory the kernels write through its device alias: the active
// count by the ordered selection (its count word), the rest by k_cloud_mirror
enum
{
    DSM_PUB_N_ACTIVE,     // points the ordered selection wrote to the active buffer
    DSM_PUB_N_INACTIVE,   // store size at the snapshot
    DSM_PUB_PREV,         // store size at the previous snapshot
    DSM_PUB_CHANGED_FROM, // lowest index below the size whose point differs from the previous snapshot, else the size
    DSM_PUB_CHUNKS,       // chunks forwarded to the host mirror
    DSM_PUB_ERR_TAG,      // the sticky error word of dsm_fuse_stream_window at the snapshot, and
    DSM_PUB_ERR_FRAME,    // the frame it rejected
    DSM_PUB_WORDS
};
#define DSM_PUB_CHUNK 256 // points per CTA of k_cloud_mirror: the unit compared with the shadow and forwarded
// The inactive cloud into its host mirror, changed chunks only (k_cloud_mirror).  store == nullptr: no store, size 0.
// size_word: the store size on the device; res: the resident offsets with the error word; `upper` >= size sizes the
// grid; state: device [4], {0, INT_MAX, 0, 0} when the shadow is new
void dsm_launch_cloud_mirror(const dsm_surfel_t *store, const int32_t *size_word, const int32_t *res, int upper, float4 *shadow,
                             float4 *mirror, int32_t *state, int32_t *header, cudaStream_t s);

// Image of dsm_checkpoint_enqueue, written by k_map_snapshot on the context's stream and copied by k_map_drain into its
// pinned host twin: a 128-byte header line of DSM_SNAP_* words, then the pool (slot order), the store (store order) and
// the segment table packed to int32 (keyframe, offset, count), each section at a 128-byte aligned offset and sized for
// its capacity.  The file's writer stitches the sections together (DESIGN.md §8.5).
enum
{
    DSM_SNAP_N_POOL,     // res_ofs[1] at the snapshot
    DSM_SNAP_N_STORE,    // win_hdr[0] (0 without a store)
    DSM_SNAP_N_SEGMENTS, // win_hdr[1] (0 without a store)
    DSM_SNAP_ERR_TAG,    // the sticky error word of dsm_fuse_stream_window, and
    DSM_SNAP_ERR_FRAME,  // the frame it rejected
    DSM_SNAP_WORDS
};
struct DsmSnapLayout
{
    size_t pool, store, table, bytes; // byte offsets of the sections, total size
};
inline size_t dsm_line_up(size_t b) { return (b + 127) / 128 * 128; }
inline DsmSnapLayout dsm_snap_layout(int pool_cap, int store_cap)
{
    DsmSnapLayout l;
    l.pool = 128;
    l.store = l.pool + dsm_line_up((size_t)pool_cap * sizeof(dsm_surfel_t));
    l.table = l.store + dsm_line_up((size_t)store_cap * sizeof(dsm_surfel_t));
    l.bytes = l.table + dsm_line_up((size_t)store_cap * 12);
    return l;
}
// k_map_snapshot: pool_upper / store_upper >= the live sizes size the grid (surplus CTAs exit at once).  store == nullptr:
// no store, n_store = n_segments = 0.  res: {0, pool size, error tag, rejected frame}; hdr: {store size, segments, ...}
void dsm_launch_map_snapshot(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, const dsm_surfel_t *store, const int4 *seg,
                             const int32_t *hdr, int store_upper, uint8_t *image, const DsmSnapLayout &lay, cudaStream_t s);
// k_map_drain: the image's live lines (as its header gives them) to host_dev, the device alias of the pinned host image,
// on a fixed grid of `ctas` CTAs
#define DSM_DRAIN_CTAS 8
void dsm_launch_map_drain(const uint8_t *image, uint8_t *host_dev, const DsmSnapLayout &lay, int ctas, cudaStream_t s);

// dsm_checkpoint_enqueue_incremental (DESIGN.md §8.6) keeps the same image, with one flag byte per 256-surfel chunk after
// it: at lay.bytes, pool_chunks flags for the pool, then store_chunks for the store (one per chunk of each capacity).
// k_map_delta adds these words to the header line; DSM_DELTA_DONE is 0 between passes (the image's header line starts
// zeroed, and k_map_snapshot leaves these words alone).
enum
{
    DSM_DELTA_PREV_POOL = DSM_SNAP_WORDS, // the image's pool size before the pass, and
    DSM_DELTA_PREV_STORE,                 // its store size
    DSM_DELTA_DONE,                       // CTAs of the pass that have finished
    DSM_DELTA_WORDS
};
#define DSM_SNAP_CHUNK 256
inline int dsm_snap_chunks(int cap) { return (cap + DSM_SNAP_CHUNK - 1) / DSM_SNAP_CHUNK; }
// k_map_delta: k_map_snapshot's grid and chunks, written only where the live map differs from the image (or reaches beyond
// the image's size of the section); every live CTA sets its chunk's flag to 1 if it wrote it, else 0.  The table and the
// header are written whole.
void dsm_launch_map_delta(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, const dsm_surfel_t *store, const int4 *seg,
                          const int32_t *hdr, int store_upper, uint8_t *image, const DsmSnapLayout &lay, int pool_chunks, cudaStream_t s);
// k_map_drain_delta: the header line, the flag lines, the live table lines and the live lines of the flagged chunks only
void dsm_launch_map_drain_delta(const uint8_t *image, uint8_t *host_dev, const DsmSnapLayout &lay, int pool_chunks, int store_chunks,
                                int ctas, cudaStream_t s);

// dsm_field_* (DESIGN.md §8.7), dsm_field.cu.  The grid of one request: voxel edge, size, integer origin o and its fp32
// bounds lo = (float)o, hi = (float)(o + n), exact below 2^24.  The distance grid [nz][ny][nx] (int32 squared distances
// until the last pass, then fp32 distances) is followed, at word dsm_field_header(voxels), by DSM_FIELD_WORDS header
// words; one copy moves both to the host.
struct DsmFieldGrid
{
    float voxel;
    int n[3], o[3];
    float lo[3], hi[3];
};
enum
{
    DSM_FIELD_N_OCCUPIED, // occupied voxels (zeroed before the request; k_field_rows adds)
    DSM_FIELD_ERR_TAG,    // the sticky error word of dsm_fuse_stream_window at the request, and
    DSM_FIELD_ERR_FRAME,  // the frame it rejected
    DSM_FIELD_N_FREE,     // a known request: free voxels (zeroed before it; k_field_rows<true> adds)
    // a known request's query view: the three words above as a query reads them, with the count of sites (voxels that
    // are not free) in place of the occupied count, so that a query's "no site" rule holds for either kind of field
    DSM_FIELD_VIEW,
    DSM_FIELD_WORDS = DSM_FIELD_VIEW + 3
};
// voxel states of a known request's grid (the occupancy grid, carved in place)
enum
{
    DSM_STATE_UNKNOWN = 0,
    DSM_STATE_OCCUPIED = 1,
    DSM_STATE_FREE = 2
};
// The signed grid (dsm_field_signed_enable, DESIGN.md §8.16): [nz][ny][nx] like the distance grid, with its own header
// words at dsm_field_header(voxels), laid out as a query reads a field header, and the count of F after them
enum
{
    DSM_SIGNED_N_SITES,   // the request's sites (its query view's count; k_field_lines_signed copies it)
    DSM_SIGNED_ERR_TAG,   // the request's error words, copied by k_field_lines_signed
    DSM_SIGNED_ERR_FRAME,
    DSM_SIGNED_N_F,       // the voxels that are not sites (zeroed before the request; k_field_rows<KNOWN, true> adds)
    DSM_SIGNED_WORDS
};
static_assert(DSM_SIGNED_N_SITES == DSM_FIELD_N_OCCUPIED && DSM_SIGNED_ERR_TAG == DSM_FIELD_ERR_TAG &&
                  DSM_SIGNED_ERR_FRAME == DSM_FIELD_ERR_FRAME,
              "a query reads the signed header as a field header");
inline size_t dsm_field_header(size_t voxels) { return (voxels + 3) / 4 * 4; }
// traversable (DESIGN.md §8.11): free, and the stored fp32 distance at least radius
__device__ __forceinline__ bool dsm_traversable(const uint8_t *state, const int32_t *dist, int i, float radius)
{
    return state[i] == DSM_STATE_FREE && __int_as_float(dist[i]) >= radius;
}
// The point query of include/dsm.h on a distance or signed grid (DESIGN.md §8.8, §8.16): fp64 addressing, fp32
// interpolation with one rounding per operation.  Shared by k_field_query, k_field_clearance and k_trajectory.
__device__ __forceinline__ float q_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// one axis of the addressing: false outside (NaN included); else the lower and upper corner and the fraction
__device__ __forceinline__ bool q_axis(double p, double v, int o, int n, int &i, int &j, float &t)
{
    const double u = p / v - (double)o - 0.5;
    if (!(u >= 0.0 && u <= (double)(n - 1))) return false;
    i = min((int)floor(u), max(n - 2, 0));
    j = min(i + 1, n - 1);
    t = (float)(u - (double)i);
    return true;
}

// the point query at p: dist (and, with GRAD, the gradient) per include/dsm.h; inside = the point is inside the grid;
// empty: every inside point gets dist = fill and a zero gradient
template <bool GRAD>
__device__ __forceinline__ float4 q_sample(const float *__restrict__ dist, const DsmFieldGrid &g, bool empty, float fill, double px, double py,
                                           double pz, bool &inside)
{
    const double v = (double)g.voxel;
    int ix, jx, iy, jy, iz, jz;
    float tx, ty, tz;
    inside = q_axis(px, v, g.o[0], g.n[0], ix, jx, tx) && q_axis(py, v, g.o[1], g.n[1], iy, jy, ty) && q_axis(pz, v, g.o[2], g.n[2], iz, jz, tz);
    if (!inside) return make_float4(__int_as_float(0x7fc00000), 0.f, 0.f, 0.f);
    if (empty) return make_float4(fill, 0.f, 0.f, 0.f);
    const size_t nx = (size_t)g.n[0], ny = (size_t)g.n[1];
    const size_t r00 = (iz * ny + iy) * nx, r10 = (iz * ny + jy) * nx, r01 = (jz * ny + iy) * nx, r11 = (jz * ny + jy) * nx;
    const float c000 = __ldg(dist + r00 + ix), c100 = __ldg(dist + r00 + jx), c010 = __ldg(dist + r10 + ix), c110 = __ldg(dist + r10 + jx);
    const float c001 = __ldg(dist + r01 + ix), c101 = __ldg(dist + r01 + jx), c011 = __ldg(dist + r11 + ix), c111 = __ldg(dist + r11 + jx);
    float4 r;
    r.x = q_lerp(q_lerp(q_lerp(c000, c100, tx), q_lerp(c010, c110, tx), ty), q_lerp(q_lerp(c001, c101, tx), q_lerp(c011, c111, tx), ty), tz);
    if (GRAD)
    {
        r.y = __fdiv_rn(q_lerp(q_lerp(__fsub_rn(c100, c000), __fsub_rn(c110, c010), ty), q_lerp(__fsub_rn(c101, c001), __fsub_rn(c111, c011), ty), tz), g.voxel);
        r.z = __fdiv_rn(q_lerp(q_lerp(__fsub_rn(c010, c000), __fsub_rn(c110, c100), tx), q_lerp(__fsub_rn(c011, c001), __fsub_rn(c111, c101), tx), tz), g.voxel);
        r.w = __fdiv_rn(q_lerp(q_lerp(__fsub_rn(c001, c000), __fsub_rn(c101, c100), tx), q_lerp(__fsub_rn(c011, c010), __fsub_rn(c111, c110), tx), ty), g.voxel);
    }
    else
        r.y = r.z = r.w = 0.f;
    return r;
}

// the rules of a field without a site (+inf) and, SIGNED, of one without a voxel of F (-inf): whether one applies, and
// the distance it gives
template <bool SIGNED>
__device__ __forceinline__ bool q_empty(const int32_t *__restrict__ fhdr, float &fill)
{
    const bool no_site = fhdr[DSM_FIELD_N_OCCUPIED] == 0;
    fill = SIGNED && !no_site ? -INFINITY : INFINITY;
    return no_site || (SIGNED && fhdr[DSM_SIGNED_N_F] == 0);
}
int dsm_field_setup(); // raises the dynamic shared-memory limit of the envelope passes (lines of up to 1024 voxels)
// k_field_mark over pool slots [0, res[1]) with update_times >= min_update_times and stored surfels [0, *store_size);
// pool_upper / store_upper >= the live sizes size the grid.  store == nullptr: no store.  occ must be zeroed.
void dsm_launch_field_mark(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, int min_update_times, const dsm_surfel_t *store,
                           const int32_t *store_size, int store_upper, const DsmFieldGrid &g, uint8_t *occ, int32_t *header, cudaStream_t s);
// the three EDT passes: occ -> dist (in place from the second pass on); header[DSM_FIELD_N_OCCUPIED] must be zeroed.
// known: occ holds voxel states, the sites are the voxels that are not free, and header[DSM_FIELD_N_FREE] and
// header[DSM_FIELD_VIEW] must be zeroed as well.  sdist != nullptr: then the signed grid's three passes into sdist, whose
// header (at dsm_field_header(voxels)) must have DSM_SIGNED_N_F zeroed
void dsm_launch_field_edt(const DsmFieldGrid &g, const uint8_t *occ, bool known, int32_t *dist, int32_t *header, int32_t *sdist, cudaStream_t s);
// dsm_views_capture: the rays of one frame slot's S seeds from its plane rows (plane = d.plane + slot * S * 3)
void dsm_launch_views_capture(const float4 *plane, int S, float4 *rays, cudaStream_t s);
// k_field_carve's CTAs per view, and the most views one launch takes: the grid is one-dimensional, n_views * per_view
// CTAs, below 2^31
#define CARVE_BLOCK 128
inline int dsm_carve_ctas_per_view(int S) { return (S + CARVE_BLOCK - 1) / CARVE_BLOCK; }
// k_field_carve over n_views views of S rays each: view j reads the rays of slot slots[j] and the pose poses[12 j ..]
// (row-major [R | t], camera to world); occ must hold the marks of k_field_mark.  No launch for n_views == 0.
void dsm_launch_field_carve(const DsmFieldGrid &g, const float4 *rays, int S, const double *poses, const int32_t *slots, int n_views,
                            float max_range, uint8_t *occ, cudaStream_t s);

// dsm_frontier_* (DESIGN.md §8.10), dsm_frontier.cu.  One packed result (D2H), which the reach, gain and viewpoint jobs
// read on the device as well (DsmFrontier::table_at, list_at):
//   int32 header[DSM_FRONTIER_WORDS] | dsm_frontier_cluster_t table[max_clusters] | int32 list[max_voxels]
enum
{
    DSM_FRONTIER_N_FRONTIER, // the four words of dsm_frontier_counts_t, zeroed before the job
    DSM_FRONTIER_N_COMPONENTS,
    DSM_FRONTIER_N_CLUSTERS,
    DSM_FRONTIER_N_LISTED,
    DSM_FRONTIER_ERR_TAG,    // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_frontier_mark
    DSM_FRONTIER_ERR_FRAME,
    DSM_FRONTIER_N_LISTED_CLUSTERS, // scratch: the table entries whose voxels are in the list
    DSM_FRONTIER_N_SELECTED,        // scratch: the members the list compaction selected
    DSM_FRONTIER_WORDS = 8          // 32 B: the table stays 8-byte aligned
};
// the frontier table's cluster among the first n whose listed members hold list entry j, or -1 (a binary search over
// the offsets: the listed clusters are a prefix of the table with rising offsets)
__device__ __forceinline__ int dsm_frontier_cluster_of(const dsm_frontier_cluster_t *table, int n, int j)
{
    int lo = 0, hi = n; // the last c with offset in [0, j]
    while (lo < hi)
    {
        const int m = (lo + hi) / 2;
        const int o = table[m].offset;
        if (o >= 0 && o <= j)
            lo = m + 1;
        else
            hi = m;
    }
    const int c = lo - 1;
    return c >= 0 && j < table[c].offset + table[c].n_voxels ? c : -1;
}

// dsm_gain_* (DESIGN.md §8.12), dsm_gain.cu, and what the viewpoint and heading jobs share with it: one view as the host
// stages it (the pose, its box of grid voxels (lo, size; size 0 on an axis: empty), the named cluster (-1) and the
// view's first brick in the launch), the bricks, the frustum test and the line of sight
struct DsmGainView
{
    double P[12];
    int32_t lo[3], size[3], cluster, brick0;
}; // 128 B
#define DSM_GAIN_BX 8 // bricks of 8 x 8 x 4 voxels, one CTA of 256 threads each
#define DSM_GAIN_BY 8
#define DSM_GAIN_BZ 4
inline long long dsm_gain_bricks(const int32_t size[3])
{
    return (long long)((size[0] + DSM_GAIN_BX - 1) / DSM_GAIN_BX) * ((size[1] + DSM_GAIN_BY - 1) / DSM_GAIN_BY) *
           ((size[2] + DSM_GAIN_BZ - 1) / DSM_GAIN_BZ);
}
// Gain's frustum test (include/dsm.h) of d = c - t for the camera-to-world rotation R_km = R[S k + m] (S = 4: a
// pose's 3x4 rows, S = 3: a bare rotation); every step fp64 with one rounding.  Shared by k_gain_views and
// k_vp_score.
template <int S>
__device__ __forceinline__ bool dsm_gain_frustum(const double *R, double d0, double d1, double d2, double fx, double fy, double cx,
                                                 double cy, double width, double height, double range2)
{
    const double r2 = __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
    const double qz = __dadd_rn(__dadd_rn(__dmul_rn(R[2], d0), __dmul_rn(R[S + 2], d1)), __dmul_rn(R[2 * S + 2], d2));
    if (!(r2 <= range2 && qz > 0.0)) return false;
    const double qx = __dadd_rn(__dadd_rn(__dmul_rn(R[0], d0), __dmul_rn(R[S], d1)), __dmul_rn(R[2 * S], d2));
    const double qy = __dadd_rn(__dadd_rn(__dmul_rn(R[1], d0), __dmul_rn(R[S + 1], d1)), __dmul_rn(R[2 * S + 1], d2));
    const double u = __dadd_rn(__dmul_rn(fx, __ddiv_rn(qx, qz)), cx), w = __dadd_rn(__dmul_rn(fy, __ddiv_rn(qy, qz)), cy);
    return u >= 0.0 && u < width && w >= 0.0 && w < height;
}
// Gain's line of sight (include/dsm.h): the walk from a = t to b = c (both fp64 world points within max_range of each
// other, so every index stays within int) reaches floor(c / v), each voxel before it inside the grid and passing the
// blocking rule; it leaves at the first voxel that does not.  Shared by k_gain_views and k_vp_score.
__device__ __forceinline__ bool dsm_gain_walk(const DsmFieldGrid &g, const uint8_t *__restrict__ state, int unknown_blocks, double tx,
                                              double ty, double tz, double c0, double c1, double c2)
{
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const double v = (double)g.voxel;
    const double wa0 = __ddiv_rn(tx, v), wa1 = __ddiv_rn(ty, v), wa2 = __ddiv_rn(tz, v);
    const double wb0 = __ddiv_rn(c0, v), wb1 = __ddiv_rn(c1, v), wb2 = __ddiv_rn(c2, v);
    int ix = (int)floor(wa0), iy = (int)floor(wa1), iz = (int)floor(wa2);
    const int ex = (int)floor(wb0), ey = (int)floor(wb1), ez = (int)floor(wb2);
    const double e0 = __dsub_rn(wb0, wa0), e1 = __dsub_rn(wb1, wa1), e2 = __dsub_rn(wb2, wa2);
    const int s0 = e0 > 0.0 ? 1 : (e0 < 0.0 ? -1 : 0), s1 = e1 > 0.0 ? 1 : (e1 < 0.0 ? -1 : 0), s2 = e2 > 0.0 ? 1 : (e2 < 0.0 ? -1 : 0);
    const double D0 = s0 != 0 ? __drcp_rn(fabs(e0)) : INFINITY, D1 = s1 != 0 ? __drcp_rn(fabs(e1)) : INFINITY,
                 D2 = s2 != 0 ? __drcp_rn(fabs(e2)) : INFINITY;
    double mx = s0 != 0 ? __ddiv_rn(__dsub_rn((double)(s0 > 0 ? ix + 1 : ix), wa0), e0) : INFINITY;
    double my = s1 != 0 ? __ddiv_rn(__dsub_rn((double)(s1 > 0 ? iy + 1 : iy), wa1), e1) : INFINITY;
    double mz = s2 != 0 ? __ddiv_rn(__dsub_rn((double)(s2 > 0 ? iz + 1 : iz), wa2), e2) : INFINITY;
    while (true)
    {
        if (ix == ex && iy == ey && iz == ez) return true;
        const int px = ix - g.o[0], py = iy - g.o[1], pz = iz - g.o[2];
        if (!((unsigned)px < (unsigned)nx && (unsigned)py < (unsigned)ny && (unsigned)pz < (unsigned)nz)) return false;
        const uint8_t s = __ldg(state + ((size_t)pz * ny + py) * nx + px);
        if (unknown_blocks ? s != DSM_STATE_FREE : s == DSM_STATE_OCCUPIED) return false;
        // argmin, the lowest axis on ties
        if (mx <= my && mx <= mz)
        {
            if (mx > 1.0) return false;
            ix += s0;
            mx = __dadd_rn(mx, D0);
        }
        else if (my <= mz)
        {
            if (my > 1.0) return false;
            iy += s1;
            my = __dadd_rn(my, D1);
        }
        else
        {
            if (mz > 1.0) return false;
            iz += s2;
            mz = __dadd_rn(mz, D2);
        }
    }
}
