// Wire formats on the output side of the hot path (SURVEY.md §8f row 4): the two files the reference's
// ~save_map callback writes (ros_node.cpp -> SurfelMap::save_cloud / save_mesh).  Host code only — text
// formatting is not GPU work; the device part is the filtered, ordered export of the resident pool
// (dsm_pool_export_cloud / dsm_pool_export_surfels in dsm_capi.cu).
//
//  dsm_write_pcd       pcl::io::savePCDFile(name, cloud) as called at surfel_map.cpp:1171 for a
//                      pcl::PointCloud<pcl::PointXYZI>: PCD v0.7, fields x y z intensity, one float each.
//                      PCL is a third-party dependency that is not vendored in the reference tree; the layout
//                      below restates its published PCD v0.7 writer (ASCII: 8 significant digits, "nan" for NaN,
//                      single spaces, '\n' line ends; binary: the packed 16-byte records after "DATA binary").
//  dsm_write_ply_mesh  SurfelMap::save_mesh (surfel_map.cpp:1229-1280) with push_a_surfel (:1175-1226): every
//                      surfel becomes a hexagon of 6 vertices (grey colour) and 4 triangles, ASCII PLY, numbers
//                      in the default ostream format (%g), each vertex value followed by one space.
//  dsm_map_save        the checkpoint of the GPU-resident map (DESIGN.md §8.4), and its readers dsm_map_load /
//  dsm_map_load        dsm_map_peek.  This file alone knows the layout; all fields little-endian:
//  dsm_map_peek          0  char magic[8] "DSMMAP\0\0"    8  uint32 format version    12  int32 dsm_version()
//                       16  int32 W, H    24  float fx, fy, cx, cy, far, near    48  double the four dsm_constants
//                       80  int32 n_pool, n_store, n_segments, 0    96  uint64 extra_bytes
//                      104  dsm_surfel_t pool[n_pool] (slot order), dsm_surfel_t store[n_store] (store order),
//                           int32 table[n_segments][3] (keyframe, offset, count), uint8 extra[extra_bytes],
//                           uint64 FNV-1a 64 of every byte before it
//                      dsm_map_write is the one writer of that file: dsm_map_save and the checkpoint thread of
//                      dsm_checkpoint_enqueue (dsm_capi.cu) hand it the header fields and the sections as spans.
//                      Version 2, of a context after dsm_checkpoint_views_enable (DESIGN.md §8.18): the word at 92 holds
//                      S, the rays per view, which must be (W/8)·(H/8); after the table come int32 n_views,
//                      int32 slots[n_views] (strictly ascending, >= 0) and float4 rays[n_views][S], then extra and the
//                      checksum as in version 1.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/dsm.h"
#include "dsm_map_state.h"

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "the checkpoint file is written in host byte order, which must be little-endian"
#endif

namespace
{
struct File
{
    FILE *f;
    explicit File(const char *path) : f(std::fopen(path, "wb")) {}
    ~File()
    {
        if (f) std::fclose(f);
    }
    bool close()
    {
        const bool ok = f && std::fflush(f) == 0 && !std::ferror(f);
        if (f) std::fclose(f);
        f = nullptr;
        return ok;
    }
};

// one PCD ASCII value: ostream << float at precision 8, NaN spelled "nan" whatever its sign
inline int put_pcd_value(char *dst, float v)
{
    if (std::isnan(v))
    {
        std::memcpy(dst, "nan", 3);
        return 3;
    }
    return std::snprintf(dst, 32, "%.8g", (double)v);
}

// push_a_surfel (surfel_map.cpp:1175-1226): 6 vertices x (x, y, z, c, c, c); float arithmetic in the
// reference's operation order (this file is built with -ffp-contract=off)
void hexagon(const dsm_surfel_t &e, float *v)
{
    const float c = (float)(int)e.color; // "int surfel_color = this_surfel.color" (:1177), pushed back as float
    const float px = e.px, py = e.py, pz = e.pz;
    float xd[3] = {-1 * e.ny, e.nx, 0.f}; // :1186-1188
    {                                     // x_dir.normalize() (:1189): Eigen leaves a zero vector untouched
        const float z = xd[0] * xd[0] + xd[1] * xd[1] + xd[2] * xd[2];
        if (z > 0.f)
        {
            const float n = std::sqrt(z);
            xd[0] /= n, xd[1] /= n, xd[2] /= n;
        }
    }
    const float yd[3] = {e.ny * xd[2] - e.nz * xd[1], e.nz * xd[0] - e.nx * xd[2], e.nx * xd[1] - e.ny * xd[0]}; // :1191
    const float radius = e.size;
    const float h_r = (float)((double)radius * 0.5);     // :1193
    const float t_r = (float)((double)radius * 0.86603); // :1194
    const float p[3] = {px, py, pz};
    const float sx[6] = {-h_r, h_r, -radius, radius, -h_r, h_r}; // :1196-1201
    const float sy[6] = {-t_r, -t_r, 0.f, 0.f, t_r, t_r};
    for (int k = 0; k < 6; k++)
    {
        for (int a = 0; a < 3; a++)
        {
            float q = p[a] + xd[a] * sx[k]; // p -/+ x_dir * r  (x*(-r) == -(x*r) exactly)
            if (k != 2 && k != 3) q = q + yd[a] * sy[k];
            v[k * 6 + a] = q;
        }
        v[k * 6 + 3] = v[k * 6 + 4] = v[k * 6 + 5] = c;
    }
}
} // namespace

extern "C" int dsm_write_pcd(const char *path, const dsm_point_t *pts, size_t n, int binary)
{
    if (!path || (n > 0 && !pts)) return DSM_E_INVALID;
    File out(path);
    if (!out.f) return DSM_E_IO;
    std::fprintf(out.f,
                 "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\n"
                 "TYPE F F F F\nCOUNT 1 1 1 1\nWIDTH %zu\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %zu\nDATA %s\n",
                 n, n, binary ? "binary" : "ascii");
    if (binary)
    {
        if (n > 0 && std::fwrite(pts, sizeof(dsm_point_t), n, out.f) != n) return DSM_E_IO;
    }
    else
    {
        char line[160];
        for (size_t i = 0; i < n; i++)
        {
            const float v[4] = {pts[i].x, pts[i].y, pts[i].z, pts[i].intensity};
            int len = 0;
            for (int k = 0; k < 4; k++)
            {
                len += put_pcd_value(line + len, v[k]);
                line[len++] = k < 3 ? ' ' : '\n';
            }
            if (std::fwrite(line, 1, (size_t)len, out.f) != (size_t)len) return DSM_E_IO;
        }
    }
    return out.close() ? DSM_OK : DSM_E_IO;
}

extern "C" int dsm_mesh_vertices(const dsm_surfel_t *surfels, size_t n, float *vertices36)
{
    if (n > 0 && (!surfels || !vertices36)) return DSM_E_INVALID;
    for (size_t i = 0; i < n; i++) hexagon(surfels[i], vertices36 + i * 36);
    return DSM_OK;
}

extern "C" int dsm_write_ply_mesh(const char *path, const dsm_surfel_t *surfels, size_t n)
{
    if (!path || (n > 0 && !surfels)) return DSM_E_INVALID;
    File out(path);
    if (!out.f) return DSM_E_IO; // the reference returns silently when the stream cannot be opened (:1232-1233)
    std::fprintf(out.f,
                 "ply\nformat ascii 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %zu\n"
                 "property list uchar int vertex_index\nend_header\n",
                 n * 6, n * 4);
    float v[36];
    char line[6 * 24 + 8];
    for (size_t i = 0; i < n; i++)
    {
        hexagon(surfels[i], v);
        for (int k = 0; k < 6; k++)
        {
            int len = 0;
            for (int j = 0; j < 6; j++)
            {
                len += std::snprintf(line + len, 24, "%g", (double)v[k * 6 + j]);
                line[len++] = ' ';
            }
            line[len++] = '\n';
            if (std::fwrite(line, 1, (size_t)len, out.f) != (size_t)len) return DSM_E_IO;
        }
    }
    for (size_t i = 0; i < n; i++)
    { // :1266-1278
        const size_t p1 = i * 6, p2 = p1 + 1, p3 = p1 + 2, p4 = p1 + 3, p5 = p1 + 4, p6 = p1 + 5;
        std::fprintf(out.f, "3 %zu %zu %zu\n3 %zu %zu %zu\n3 %zu %zu %zu\n3 %zu %zu %zu\n", p1, p2, p3, p2, p4, p3, p3, p4, p5,
                     p5, p4, p6);
    }
    return out.close() ? DSM_OK : DSM_E_IO;
}

// ---- checkpoint of the GPU-resident map ----
namespace
{
const char kMapMagic[8] = {'D', 'S', 'M', 'M', 'A', 'P', 0, 0};
const uint32_t kMapFormat = 1, kMapFormatViews = 2;

struct MapHeader // the first 104 bytes of the file, in file order
{
    char magic[8];
    uint32_t format;
    int32_t version;
    int32_t width, height;
    float fx, fy, cx, cy, fuse_far, fuse_near;
    dsm_constants constants;
    int32_t n_pool, n_store, n_segments, rays_per_view; // rays_per_view: 0 in version 1
    uint64_t extra_bytes;
};
static_assert(sizeof(MapHeader) == 104, "checkpoint header layout");

struct Fnv1a
{
    uint64_t h = 14695981039346656037ull;
    void add(const void *p, size_t n)
    {
        const uint8_t *b = static_cast<const uint8_t *>(p);
        for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
    }
};

// A whole file into `raw`: DSM_E_IO if it cannot be opened or read
int read_all(const char *path, std::vector<uint8_t> &raw)
{
    FILE *f = std::fopen(path, "rb");
    if (!f) return DSM_E_IO;
    long len = -1;
    if (std::fseek(f, 0, SEEK_END) == 0) len = std::ftell(f);
    if (len >= 0 && std::fseek(f, 0, SEEK_SET) == 0)
    {
        raw.resize((size_t)len);
        if (len > 0 && std::fread(raw.data(), 1, (size_t)len, f) != (size_t)len) len = -1;
    }
    std::fclose(f);
    return len < 0 ? DSM_E_IO : DSM_OK;
}

// The rays per view of a version-2 header: dsm_num_seeds of its frame size
int64_t seeds_of(const MapHeader &h) { return (int64_t)(h.width / 8) * (h.height / 8); }

bool ascending(const int32_t *slots, int64_t n)
{
    for (int64_t i = 0; i < n; i++)
        if (slots[i] < 0 || (i > 0 && slots[i] <= slots[i - 1])) return false;
    return true;
}

// A checkpoint read whole and checked: magic, version and, in version 2, the rays-per-view word (DSM_E_INVALID), then
// its length and checksum (DSM_E_IO), then the views section's slot list (DSM_E_INVALID)
struct MapFile
{
    std::vector<uint8_t> raw;
    MapHeader hdr;
    const dsm_surfel_t *pool = nullptr, *store = nullptr;
    const int32_t *table = nullptr;
    const uint8_t *extra = nullptr;
    int rays_per_view = 0, n_views = 0; // 0 and 0 in version 1
    const int32_t *view_slots = nullptr;
    const uint8_t *view_rays = nullptr; // [n_views][rays_per_view] float4

    int read(const char *path)
    {
        const int rc = read_all(path, raw);
        return rc != DSM_OK ? rc : parse();
    }
    // the checks of read() on the bytes in `raw`
    int parse()
    {
        if (raw.size() < 16) return DSM_E_IO;
        std::memcpy(&hdr, raw.data(), std::min(raw.size(), sizeof(hdr)));
        if (std::memcmp(hdr.magic, kMapMagic, 8) != 0 || (hdr.format != kMapFormat && hdr.format != kMapFormatViews))
            return DSM_E_INVALID;
        if (raw.size() < sizeof(hdr) + 8) return DSM_E_IO;
        const bool views = hdr.format == kMapFormatViews;
        if (views && (hdr.rays_per_view < 1 || hdr.rays_per_view != seeds_of(hdr))) return DSM_E_INVALID;
        if (hdr.n_pool < 0 || hdr.n_store < 0 || hdr.n_segments < 0) return DSM_E_IO;
        uint64_t body = (uint64_t)(hdr.n_pool + (uint64_t)hdr.n_store) * sizeof(dsm_surfel_t) + (uint64_t)hdr.n_segments * 12;
        int32_t nv = 0;
        if (views)
        {
            if (body > raw.size() || sizeof(hdr) + body + 4 + 8 > raw.size()) return DSM_E_IO;
            std::memcpy(&nv, raw.data() + sizeof(hdr) + body, 4);
            if (nv < 0 || (nv > 0 && (uint64_t)hdr.rays_per_view > raw.size() / 16 / (uint64_t)nv)) return DSM_E_IO;
            body += 4 + 4 * (uint64_t)nv + 16 * (uint64_t)hdr.rays_per_view * (uint64_t)nv;
        }
        if (hdr.extra_bytes > raw.size() || body > raw.size() || sizeof(hdr) + body + hdr.extra_bytes + 8 != raw.size()) return DSM_E_IO;
        Fnv1a sum;
        sum.add(raw.data(), raw.size() - 8);
        uint64_t want = 0;
        std::memcpy(&want, raw.data() + raw.size() - 8, 8);
        if (sum.h != want) return DSM_E_IO;
        const uint8_t *p = raw.data() + sizeof(hdr);
        pool = reinterpret_cast<const dsm_surfel_t *>(p);
        store = pool + hdr.n_pool;
        table = reinterpret_cast<const int32_t *>(store + hdr.n_store);
        extra = reinterpret_cast<const uint8_t *>(table + 3 * (size_t)hdr.n_segments);
        rays_per_view = views ? hdr.rays_per_view : 0;
        n_views = nv;
        if (views)
        {
            view_slots = reinterpret_cast<const int32_t *>(extra) + 1;
            view_rays = reinterpret_cast<const uint8_t *>(view_slots + nv);
            extra = view_rays + 16 * (size_t)hdr.rays_per_view * nv;
            if (!ascending(view_slots, nv)) return DSM_E_INVALID;
        }
        return DSM_OK;
    }
};

// the file under a temporary name next to `path`; renamed over `path` once written and flushed to the disk
struct AtomicFile
{
    std::string path, tmp;
    FILE *f = nullptr;
    Fnv1a sum;
    uint64_t bytes = 0; // written so far
    bool ok = true, created = false, renamed = false;

    explicit AtomicFile(const char *p) : path(p), tmp(std::string(p) + ".tmp." + std::to_string((long)getpid()))
    {
        const int fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_EXCL, 0666);
        created = fd >= 0;
        if (created) f = fdopen(fd, "wb");
        if (created && !f) ::close(fd);
        ok = f != nullptr;
    }
    ~AtomicFile()
    {
        if (f) std::fclose(f);
        if (created && !renamed) std::remove(tmp.c_str());
    }
    void put(const void *p, size_t n)
    {
        if (!ok || n == 0) return;
        sum.add(p, n);
        ok = std::fwrite(p, 1, n, f) == n;
        bytes += n;
    }
    bool commit()
    {
        const uint64_t h = sum.h;
        put(&h, 8);
        if (!f) return false; // the temporary could not be created
        ok = ok && std::fflush(f) == 0 && fsync(fileno(f)) == 0;
        ok = std::fclose(f) == 0 && ok;
        f = nullptr;
        ok = ok && std::rename(tmp.c_str(), path.c_str()) == 0;
        renamed = ok;
        if (ok)
        { // the rename itself reaches the disk with its directory
            const size_t slash = path.find_last_of('/');
            const std::string dir = slash == std::string::npos ? "." : (slash == 0 ? "/" : path.substr(0, slash));
            const int dfd = ::open(dir.c_str(), O_RDONLY);
            if (dfd >= 0)
            {
                fsync(dfd);
                ::close(dfd);
            }
        }
        return ok;
    }
};
} // namespace

extern "C" int dsm_map_save(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes)
{
    if (!ctx || !path || (extra_bytes > 0 && !extra)) return DSM_E_INVALID;
    DsmMapInfo info;
    int rc = dsm_map_info(ctx, &info);
    int n_pool = 0, n_store = 0, n_seg = 0;
    if (rc == DSM_OK) rc = dsm_pool_size(ctx, &n_pool); // DSM_E_STATE without a pool; reports a rejected frame
    std::vector<dsm_surfel_t> pool((size_t)n_pool + 1), store(1);
    std::vector<int32_t> table(3), slots;
    std::vector<uint8_t> rays;
    if (rc == DSM_OK) rc = dsm_pool_download(ctx, pool.data(), n_pool, &n_pool);
    if (rc == DSM_OK && info.store_cap > 0)
    {
        rc = dsm_inactive_size(ctx, &n_store, &n_seg);
        store.resize((size_t)n_store + 1);
        table.resize(3 * (size_t)n_seg + 3);
        if (rc == DSM_OK) rc = dsm_inactive_download(ctx, -1, store.data(), n_store, &n_store);
        if (rc == DSM_OK) rc = dsm_inactive_segments(ctx, table.data(), n_seg, &n_seg);
    }
    if (rc == DSM_OK && info.view_rays > 0) rc = dsm_views_download(ctx, slots, rays);
    if (rc != DSM_OK) return rc;
    std::vector<const void *> views(slots.size());
    for (size_t i = 0; i < slots.size(); i++) views[i] = rays.data() + 16 * (size_t)info.view_rays * i;
    return dsm_map_write(path, info, DsmMapSections{pool.data(), n_pool, store.data(), n_store, table.data(), n_seg, extra, extra_bytes,
                                                    slots.data(), (int)slots.size(), views.data(), info.view_rays});
}

int dsm_map_write(const char *path, const DsmMapInfo &info, const DsmMapSections &s, uint64_t *checksum, uint64_t *bytes)
{
    MapHeader h;
    std::memset(&h, 0, sizeof(h));
    std::memcpy(h.magic, kMapMagic, 8);
    h.format = s.rays_per_view > 0 ? kMapFormatViews : kMapFormat;
    h.version = dsm_version();
    const dsm_params &p = info.params;
    h.width = p.width, h.height = p.height;
    h.fx = p.fx, h.fy = p.fy, h.cx = p.cx, h.cy = p.cy, h.fuse_far = p.fuse_far, h.fuse_near = p.fuse_near;
    h.constants = info.constants;
    h.n_pool = s.n_pool, h.n_store = s.n_store, h.n_segments = s.n_segments, h.rays_per_view = s.rays_per_view;
    h.extra_bytes = s.extra_bytes;
    AtomicFile out(path);
    out.put(&h, sizeof(h));
    out.put(s.pool, (size_t)s.n_pool * sizeof(dsm_surfel_t));
    out.put(s.store, (size_t)s.n_store * sizeof(dsm_surfel_t));
    out.put(s.table, (size_t)s.n_segments * 12);
    if (s.rays_per_view > 0)
    {
        out.put(&s.n_views, 4);
        out.put(s.view_slots, 4 * (size_t)s.n_views);
        for (int i = 0; i < s.n_views; i++) out.put(s.view_rays[i], 16 * (size_t)s.rays_per_view);
    }
    out.put(s.extra, s.extra_bytes);
    const uint64_t sum = out.sum.h;
    if (!out.commit()) return DSM_E_IO;
    if (checksum) *checksum = sum;
    if (bytes) *bytes = out.bytes;
    return DSM_OK;
}


namespace
{
// The checks and the load of dsm_map_load on a file already read and checked
int load_checked(dsm_ctx *ctx, const DsmMapInfo &info, const MapFile &m, void *extra, size_t extra_cap, size_t *extra_bytes)
{
    const MapHeader &h = m.hdr;
    const dsm_params &p = info.params;
    const float geo[6] = {p.fx, p.fy, p.cx, p.cy, p.fuse_far, p.fuse_near};
    if (h.width != p.width || h.height != p.height || std::memcmp(&h.fx, geo, sizeof(geo)) != 0 ||
        std::memcmp(&h.constants, &info.constants, sizeof(dsm_constants)) != 0)
        return DSM_E_INVALID; // the caller sets the constants before loading
    if (h.n_pool > p.max_local_surfels) return DSM_E_CAPACITY;
    if (info.publish_in_flight || info.field_in_flight) return DSM_E_STATE;
    int rc = DSM_OK;
    if (info.store_cap == 0)
    {
        if (h.n_store > 0) return DSM_E_STATE;
        if (h.n_segments > 0) return DSM_E_INVALID;
    }
    else
    {
        rc = dsm_inactive_load_check(ctx, m.store, h.n_store, m.table, h.n_segments);
        if (rc != DSM_OK) return rc;
    }
    // views: a context that did not opt in refuses a views section, as a context without a store refuses stored surfels
    if (m.rays_per_view > 0 && info.view_rays == 0) return DSM_E_STATE;
    if (m.rays_per_view > 0)
    {
        rc = dsm_views_load_check(ctx, m.view_slots, m.n_views, m.view_rays);
        if (rc != DSM_OK) return rc;
    }
    if (extra_bytes) *extra_bytes = (size_t)h.extra_bytes;
    if (h.extra_bytes > extra_cap) return DSM_E_CAPACITY;
    dsm_checkpoint_map_replaced(ctx);
    rc = dsm_pool_upload(ctx, m.pool, h.n_pool);
    if (rc == DSM_OK && info.store_cap > 0) rc = dsm_inactive_load(ctx, m.store, h.n_store, m.table, h.n_segments);
    // a file without a views section leaves no slot filled
    if (rc == DSM_OK && info.view_rays > 0) rc = dsm_views_load(ctx, m.view_slots, m.n_views, m.view_rays);
    if (rc != DSM_OK) return rc;
    if (h.extra_bytes > 0) std::memcpy(extra, m.extra, (size_t)h.extra_bytes);
    return DSM_OK;
}

// What dsm_map_peek returns of a file already read and checked
void peek_checked(const MapFile &m, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt, int seg_cap,
                  int *n_segments)
{
    if (extra_bytes) *extra_bytes = (size_t)m.hdr.extra_bytes;
    if (n_segments) *n_segments = m.hdr.n_segments;
    if (extra_cap > 0) std::memcpy(extra, m.extra, (size_t)std::min<uint64_t>(extra_cap, m.hdr.extra_bytes));
    if (seg_cap > 0) std::memcpy(kf_ofs_cnt, m.table, (size_t)std::min(seg_cap, m.hdr.n_segments) * 12);
}
} // namespace

extern "C" int dsm_map_load(dsm_ctx *ctx, const char *path, void *extra, size_t extra_cap, size_t *extra_bytes)
{
    if (!ctx || !path || (extra_cap > 0 && !extra)) return DSM_E_INVALID;
    DsmMapInfo info;
    int rc = dsm_map_info(ctx, &info);
    MapFile m;
    if (rc == DSM_OK) rc = m.read(path);
    if (rc != DSM_OK) return rc;
    return load_checked(ctx, info, m, extra, extra_cap, extra_bytes);
}

extern "C" int dsm_map_peek(const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt, int seg_cap,
                            int *n_segments)
{
    if (!path || (extra_cap > 0 && !extra) || seg_cap < 0 || (seg_cap > 0 && !kf_ofs_cnt)) return DSM_E_INVALID;
    MapFile m;
    const int rc = m.read(path);
    if (rc != DSM_OK) return rc;
    peek_checked(m, extra, extra_cap, extra_bytes, kf_ofs_cnt, seg_cap, n_segments);
    return DSM_OK;
}

// ---- the journal of incremental checkpoints (DESIGN.md §8.6) ----
// <path> is a version-1 or version-2 file, the base; <path>.journal holds, all fields little-endian:
//    0  char magic[8] "DSMJRNL\0"    8  uint32 format version    12  uint32 0 (S)    16  uint64 the base's trailing checksum
//   24  uint64 FNV-1a 64 of the 24 bytes before it
// then records, each:
//    0  uint64 sequence (1 for the first record after the base)    8  int32 n_pool, n_store, n_segments
//   20  int32 k_pool, k_store (chunks listed)    28  uint32 0 (k_views)    32  uint64 extra_bytes
//   40  int32 pool_chunk[k_pool], int32 store_chunk[k_store]: ascending indices of the 256-surfel chunks that changed
//       the payloads, in list order: min(256, n - 256 c) dsm_surfel_t of each chunk c (the pool's, then the store's)
//       int32 table[n_segments][3], uint8 extra[extra_bytes] (both whole)
//       uint64 the checksum of the previous record (of the base for the first)
//       uint64 FNV-1a 64 of every byte of the record before it
// A record holds every chunk that reaches beyond the previous state's size of its section.  The base is written first
// (temporary name, rename), then a fresh journal header the same way; a record is appended and flushed to the disk.
// Version 2 goes beside a version-2 base (DESIGN.md §8.18): the header word at 12 holds the base's rays per view S; a
// record's word at 28 is k_views, int32 view_slot[k_views] (strictly ascending, the slots captured since the previous
// state) follows the store's chunk list, and float4 rays[k_views][S] follow the store's payloads.  The resolved views
// are the base's with every record's slots put in, each replacing the slot's rays.
namespace
{
const char kJournalMagic[8] = {'D', 'S', 'M', 'J', 'R', 'N', 'L', 0};
const uint32_t kJournalFormat = 1, kJournalFormatViews = 2;

struct JournalHeader
{
    char magic[8];
    uint32_t format, rays_per_view; // rays_per_view: 0 in version 1
    uint64_t base_checksum;
};
static_assert(sizeof(JournalHeader) == 24, "journal header layout");

struct RecordHeader
{
    uint64_t sequence;
    int32_t n_pool, n_store, n_segments, k_pool, k_store;
    int32_t k_views; // 0 in version 1
    uint64_t extra_bytes;
};
static_assert(sizeof(RecordHeader) == 40, "journal record layout");

const int64_t kChunk = 256;
const size_t kChunkBytes = kChunk * sizeof(dsm_surfel_t);

std::string journal_path(const char *path) { return std::string(path) + ".journal"; }
int64_t chunks_of(int64_t n) { return (n + kChunk - 1) / kChunk; }
// surfels of chunk c of a section of n, 0 for a chunk outside it
int64_t chunk_count(int64_t n, int64_t c) { return c < 0 || c * kChunk >= n ? 0 : std::min(kChunk, n - c * kChunk); }

// A record's chunk list for a section of n surfels that held `prev` before it: ascending, inside the section, and
// holding every chunk that reaches beyond prev
bool list_ok(const int32_t *c, int k, int64_t n, int64_t prev)
{
    for (int i = 0; i < k; i++)
        if (c[i] < 0 || c[i] >= chunks_of(n) || (i > 0 && c[i] <= c[i - 1])) return false;
    if (n <= prev) return true;
    const int64_t need = chunks_of(n) - prev / kChunk; // chunks prev / 256 .. the last, which the list must end with
    return k >= need && c[k - need] == prev / kChunk;
}

// The one resolver: the base read and checked as dsm_map_load reads it, then the records of its journal replayed in
// order up to the first that is torn, fails its checksum, breaks the chain or is out of sequence.  m holds the file of
// the resulting state, in the base's version, parsed as a read file is.  A missing journal, or one that names another
// base, adds no record; a journal of another magic or format is DSM_E_INVALID, and so are a version-2 journal whose rays
// per view are not the base's, a journal of this base in the other version, and a complete record whose chunk or view
// lists do not describe its state.
int resolve(const char *path, MapFile &m, int *records)
{
    if (records) *records = 0;
    int rc = m.read(path);
    if (rc != DSM_OK) return rc;
    std::vector<uint8_t> j;
    if (read_all(journal_path(path).c_str(), j) != DSM_OK || j.size() < sizeof(JournalHeader) + 8) return DSM_OK;
    JournalHeader jh;
    std::memcpy(&jh, j.data(), sizeof(jh));
    if (std::memcmp(jh.magic, kJournalMagic, 8) != 0 || (jh.format != kJournalFormat && jh.format != kJournalFormatViews))
        return DSM_E_INVALID;
    const bool views = jh.format == kJournalFormatViews;
    if (views && (int64_t)jh.rays_per_view != seeds_of(m.hdr)) return DSM_E_INVALID; // never 0
    Fnv1a hs;
    hs.add(j.data(), sizeof(jh));
    uint64_t want = 0, chain = 0;
    std::memcpy(&want, j.data() + sizeof(jh), 8);
    std::memcpy(&chain, m.raw.data() + m.raw.size() - 8, 8);
    if (hs.h != want || jh.base_checksum != chain) return DSM_OK;
    if (views != (m.rays_per_view > 0)) return DSM_E_INVALID; // the journal of this base, but not of its version
    const size_t ray_bytes = 16 * (size_t)m.rays_per_view;

    MapHeader hdr = m.hdr;
    const uint8_t *mp = reinterpret_cast<const uint8_t *>(m.pool), *ms = reinterpret_cast<const uint8_t *>(m.store);
    std::vector<uint8_t> pool(mp, mp + (size_t)hdr.n_pool * sizeof(dsm_surfel_t));
    std::vector<uint8_t> store(ms, ms + (size_t)hdr.n_store * sizeof(dsm_surfel_t));
    std::vector<uint8_t> table(reinterpret_cast<const uint8_t *>(m.table), m.extra);
    std::vector<uint8_t> extra(m.extra, m.extra + hdr.extra_bytes);
    std::map<int32_t, const uint8_t *> rays; // slot -> its latest rays, in m.raw or j
    for (int i = 0; i < m.n_views; i++) rays[m.view_slots[i]] = m.view_rays + ray_bytes * i;
    std::vector<int32_t> list;
    int applied = 0;
    size_t pos = sizeof(JournalHeader) + 8;
    for (uint64_t seq = 1; pos < j.size(); seq++)
    {
        const uint8_t *p = j.data() + pos;
        const uint64_t left = j.size() - pos;
        RecordHeader r;
        if (left < sizeof(r)) break;
        std::memcpy(&r, p, sizeof(r));
        if (!views) r.k_views = 0;
        if (r.n_pool < 0 || r.n_store < 0 || r.n_segments < 0 || r.k_pool < 0 || r.k_store < 0 || r.k_views < 0) break;
        const uint64_t chunk_lists = 4 * ((uint64_t)r.k_pool + (uint64_t)r.k_store), lists = chunk_lists + 4 * (uint64_t)r.k_views;
        if (r.extra_bytes > left || sizeof(r) + lists > left) break;
        if (r.k_views > 0 && ray_bytes > left / (uint64_t)r.k_views) break; // torn
        const size_t k_chunks = (size_t)r.k_pool + r.k_store;
        list.resize(k_chunks + r.k_views);
        if (!list.empty()) std::memcpy(list.data(), p + sizeof(r), (size_t)lists);
        const int32_t *vslots = list.data() + k_chunks;
        uint64_t payload = ray_bytes * (uint64_t)r.k_views;
        for (size_t i = 0; i < k_chunks; i++)
            payload += (uint64_t)chunk_count((int)i < r.k_pool ? r.n_pool : r.n_store, list[i]) * sizeof(dsm_surfel_t);
        const uint64_t len = sizeof(r) + lists + payload + 12 * (uint64_t)r.n_segments + r.extra_bytes + 16;
        if (len > left) break; // torn
        Fnv1a s;
        s.add(p, (size_t)len - 8);
        uint64_t own = 0, prev = 0;
        std::memcpy(&prev, p + len - 16, 8);
        std::memcpy(&own, p + len - 8, 8);
        if (s.h != own || prev != chain || r.sequence != seq) break;
        if (!list_ok(list.data(), r.k_pool, r.n_pool, hdr.n_pool) || !list_ok(list.data() + r.k_pool, r.k_store, r.n_store, hdr.n_store) ||
            !ascending(vslots, r.k_views))
            return DSM_E_INVALID;
        const uint8_t *q = p + sizeof(r) + lists;
        pool.resize((size_t)r.n_pool * sizeof(dsm_surfel_t));
        store.resize((size_t)r.n_store * sizeof(dsm_surfel_t));
        for (size_t i = 0; i < k_chunks; i++)
        {
            const bool in_pool = (int)i < r.k_pool;
            const size_t n = (size_t)chunk_count(in_pool ? r.n_pool : r.n_store, list[i]) * sizeof(dsm_surfel_t);
            std::memcpy((in_pool ? pool : store).data() + (size_t)list[i] * kChunkBytes, q, n);
            q += n;
        }
        for (int i = 0; i < r.k_views; i++, q += ray_bytes) rays[vslots[i]] = q;
        table.assign(q, q + 12 * (size_t)r.n_segments);
        q += table.size();
        extra.assign(q, q + r.extra_bytes);
        hdr.n_pool = r.n_pool, hdr.n_store = r.n_store, hdr.n_segments = r.n_segments, hdr.extra_bytes = r.extra_bytes;
        chain = own;
        pos += (size_t)len;
        applied++;
    }
    if (applied == 0) return DSM_OK;
    std::vector<uint8_t> raw;
    raw.reserve(sizeof(hdr) + pool.size() + store.size() + table.size() + extra.size() + 8 +
                (views ? 4 + (4 + ray_bytes) * rays.size() : 0));
    const uint8_t *hb = reinterpret_cast<const uint8_t *>(&hdr);
    raw.insert(raw.end(), hb, hb + sizeof(hdr));
    for (const std::vector<uint8_t> *v : {&pool, &store, &table}) raw.insert(raw.end(), v->begin(), v->end());
    if (views)
    {
        const int32_t n = (int32_t)rays.size();
        const uint8_t *nb = reinterpret_cast<const uint8_t *>(&n);
        raw.insert(raw.end(), nb, nb + 4);
        for (const auto &v : rays)
        {
            const uint8_t *sb = reinterpret_cast<const uint8_t *>(&v.first);
            raw.insert(raw.end(), sb, sb + 4);
        }
        for (const auto &v : rays) raw.insert(raw.end(), v.second, v.second + ray_bytes);
    }
    raw.insert(raw.end(), extra.begin(), extra.end());
    Fnv1a sum;
    sum.add(raw.data(), raw.size());
    const uint8_t *sb = reinterpret_cast<const uint8_t *>(&sum.h);
    raw.insert(raw.end(), sb, sb + 8);
    m.raw = std::move(raw);
    rc = m.parse();
    if (rc == DSM_OK && records) *records = applied;
    return rc;
}
} // namespace

int dsm_journal_start(const char *path, uint64_t base_checksum, int rays_per_view, uint64_t *bytes)
{
    JournalHeader h;
    std::memset(&h, 0, sizeof(h));
    std::memcpy(h.magic, kJournalMagic, 8);
    h.format = rays_per_view > 0 ? kJournalFormatViews : kJournalFormat;
    h.rays_per_view = (uint32_t)std::max(rays_per_view, 0);
    h.base_checksum = base_checksum;
    AtomicFile out(journal_path(path).c_str());
    out.put(&h, sizeof(h));
    if (!out.commit()) return DSM_E_IO;
    *bytes = out.bytes;
    return DSM_OK;
}

int dsm_journal_append(const char *path, uint64_t journal_bytes, const DsmJournalRecord &r, uint64_t *checksum, uint64_t *bytes)
{
    const int fd = ::open(journal_path(path).c_str(), O_WRONLY);
    if (fd < 0) return DSM_E_IO;
    struct stat st;
    FILE *f = nullptr;
    if (fstat(fd, &st) == 0 && (uint64_t)st.st_size == journal_bytes && lseek(fd, 0, SEEK_END) >= 0) f = fdopen(fd, "wb");
    if (!f)
    { // the journal is not the one the chain ends with
        ::close(fd);
        return DSM_E_IO;
    }
    Fnv1a sum;
    uint64_t n = 0;
    bool ok = true;
    auto put = [&](const void *p, size_t len) {
        if (!ok || len == 0) return;
        sum.add(p, len);
        ok = std::fwrite(p, 1, len, f) == len;
        n += len;
    };
    RecordHeader h;
    std::memset(&h, 0, sizeof(h));
    h.sequence = r.sequence;
    h.n_pool = r.n_pool, h.n_store = r.n_store, h.n_segments = r.n_segments, h.k_pool = r.k_pool, h.k_store = r.k_store;
    h.k_views = r.k_views;
    h.extra_bytes = r.extra_bytes;
    put(&h, sizeof(h));
    put(r.pool_chunks, 4 * (size_t)r.k_pool);
    put(r.store_chunks, 4 * (size_t)r.k_store);
    put(r.view_slots, 4 * (size_t)r.k_views);
    for (int i = 0; i < r.k_pool; i++)
        put(r.pool + (size_t)r.pool_chunks[i] * kChunkBytes, (size_t)chunk_count(r.n_pool, r.pool_chunks[i]) * sizeof(dsm_surfel_t));
    for (int i = 0; i < r.k_store; i++)
        put(r.store + (size_t)r.store_chunks[i] * kChunkBytes, (size_t)chunk_count(r.n_store, r.store_chunks[i]) * sizeof(dsm_surfel_t));
    for (int i = 0; i < r.k_views; i++) put(r.view_rays[i], 16 * (size_t)r.rays_per_view);
    put(r.table, 12 * (size_t)r.n_segments);
    put(r.extra, r.extra_bytes);
    put(&r.prev_checksum, 8);
    const uint64_t own = sum.h;
    put(&own, 8);
    ok = ok && std::fflush(f) == 0 && fsync(fileno(f)) == 0;
    if (!ok && ftruncate(fileno(f), (off_t)journal_bytes) == 0) fsync(fileno(f)); // a torn tail would end every replay
    ok = std::fclose(f) == 0 && ok;
    if (!ok) return DSM_E_IO;
    *checksum = own;
    *bytes = n;
    return DSM_OK;
}

extern "C" int dsm_map_load_journal(dsm_ctx *ctx, const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int *records)
{
    if (records) *records = 0;
    if (!ctx || !path || (extra_cap > 0 && !extra)) return DSM_E_INVALID;
    DsmMapInfo info;
    int rc = dsm_map_info(ctx, &info);
    MapFile m;
    int n = 0;
    if (rc == DSM_OK) rc = resolve(path, m, &n);
    if (rc == DSM_OK) rc = load_checked(ctx, info, m, extra, extra_cap, extra_bytes);
    if (rc == DSM_OK && records) *records = n;
    return rc;
}

extern "C" int dsm_map_peek_journal(const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt,
                                    int seg_cap, int *n_segments, int *records)
{
    if (records) *records = 0;
    if (!path || (extra_cap > 0 && !extra) || seg_cap < 0 || (seg_cap > 0 && !kf_ofs_cnt)) return DSM_E_INVALID;
    MapFile m;
    const int rc = resolve(path, m, records);
    if (rc != DSM_OK) return rc;
    peek_checked(m, extra, extra_cap, extra_bytes, kf_ofs_cnt, seg_cap, n_segments);
    return DSM_OK;
}

extern "C" int dsm_journal_materialize(const char *path, const char *out_path)
{
    if (!path || !out_path) return DSM_E_INVALID;
    MapFile m;
    const int rc = resolve(path, m, nullptr);
    if (rc != DSM_OK) return rc;
    AtomicFile out(out_path);
    out.put(m.raw.data(), m.raw.size() - 8); // commit appends the same checksum
    return out.commit() ? DSM_OK : DSM_E_IO;
}
