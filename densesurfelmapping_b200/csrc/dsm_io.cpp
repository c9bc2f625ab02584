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
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
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
const uint32_t kMapFormat = 1;

struct MapHeader // the first 104 bytes of the file, in file order
{
    char magic[8];
    uint32_t format;
    int32_t version;
    int32_t width, height;
    float fx, fy, cx, cy, fuse_far, fuse_near;
    dsm_constants constants;
    int32_t n_pool, n_store, n_segments, zero;
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

// A checkpoint read whole and checked: magic and version (DSM_E_INVALID), then its length and checksum (DSM_E_IO)
struct MapFile
{
    std::vector<uint8_t> raw;
    MapHeader hdr;
    const dsm_surfel_t *pool = nullptr, *store = nullptr;
    const int32_t *table = nullptr;
    const uint8_t *extra = nullptr;

    int read(const char *path)
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
        if (len < 0) return DSM_E_IO;
        if (raw.size() < 16) return DSM_E_IO;
        std::memcpy(&hdr, raw.data(), std::min(raw.size(), sizeof(hdr)));
        if (std::memcmp(hdr.magic, kMapMagic, 8) != 0 || hdr.format != kMapFormat) return DSM_E_INVALID;
        if (raw.size() < sizeof(hdr) + 8) return DSM_E_IO;
        if (hdr.n_pool < 0 || hdr.n_store < 0 || hdr.n_segments < 0) return DSM_E_IO;
        const uint64_t body = (uint64_t)(hdr.n_pool + (uint64_t)hdr.n_store) * sizeof(dsm_surfel_t) + (uint64_t)hdr.n_segments * 12;
        if (hdr.extra_bytes > raw.size() || sizeof(hdr) + body + hdr.extra_bytes + 8 != raw.size()) return DSM_E_IO;
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
        return DSM_OK;
    }
};

// the file under a temporary name next to `path`; renamed over `path` once written and flushed to the disk
struct AtomicFile
{
    std::string path, tmp;
    FILE *f = nullptr;
    Fnv1a sum;
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
    std::vector<int32_t> table(3);
    if (rc == DSM_OK) rc = dsm_pool_download(ctx, pool.data(), n_pool, &n_pool);
    if (rc == DSM_OK && info.store_cap > 0)
    {
        rc = dsm_inactive_size(ctx, &n_store, &n_seg);
        store.resize((size_t)n_store + 1);
        table.resize(3 * (size_t)n_seg + 3);
        if (rc == DSM_OK) rc = dsm_inactive_download(ctx, -1, store.data(), n_store, &n_store);
        if (rc == DSM_OK) rc = dsm_inactive_segments(ctx, table.data(), n_seg, &n_seg);
    }
    if (rc != DSM_OK) return rc;
    return dsm_map_write(path, info, DsmMapSections{pool.data(), n_pool, store.data(), n_store, table.data(), n_seg, extra, extra_bytes});
}

int dsm_map_write(const char *path, const DsmMapInfo &info, const DsmMapSections &s)
{
    MapHeader h;
    std::memset(&h, 0, sizeof(h));
    std::memcpy(h.magic, kMapMagic, 8);
    h.format = kMapFormat;
    h.version = dsm_version();
    const dsm_params &p = info.params;
    h.width = p.width, h.height = p.height;
    h.fx = p.fx, h.fy = p.fy, h.cx = p.cx, h.cy = p.cy, h.fuse_far = p.fuse_far, h.fuse_near = p.fuse_near;
    h.constants = info.constants;
    h.n_pool = s.n_pool, h.n_store = s.n_store, h.n_segments = s.n_segments;
    h.extra_bytes = s.extra_bytes;
    AtomicFile out(path);
    out.put(&h, sizeof(h));
    out.put(s.pool, (size_t)s.n_pool * sizeof(dsm_surfel_t));
    out.put(s.store, (size_t)s.n_store * sizeof(dsm_surfel_t));
    out.put(s.table, (size_t)s.n_segments * 12);
    out.put(s.extra, s.extra_bytes);
    return out.commit() ? DSM_OK : DSM_E_IO;
}

extern "C" int dsm_map_load(dsm_ctx *ctx, const char *path, void *extra, size_t extra_cap, size_t *extra_bytes)
{
    if (!ctx || !path || (extra_cap > 0 && !extra)) return DSM_E_INVALID;
    DsmMapInfo info;
    int rc = dsm_map_info(ctx, &info);
    MapFile m;
    if (rc == DSM_OK) rc = m.read(path);
    if (rc != DSM_OK) return rc;
    const MapHeader &h = m.hdr;
    const dsm_params &p = info.params;
    const float geo[6] = {p.fx, p.fy, p.cx, p.cy, p.fuse_far, p.fuse_near};
    if (h.width != p.width || h.height != p.height || std::memcmp(&h.fx, geo, sizeof(geo)) != 0 ||
        std::memcmp(&h.constants, &info.constants, sizeof(dsm_constants)) != 0)
        return DSM_E_INVALID; // the caller sets the constants before loading
    if (h.n_pool > p.max_local_surfels) return DSM_E_CAPACITY;
    if (info.publish_in_flight) return DSM_E_STATE;
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
    if (extra_bytes) *extra_bytes = (size_t)h.extra_bytes;
    if (h.extra_bytes > extra_cap) return DSM_E_CAPACITY;
    rc = dsm_pool_upload(ctx, m.pool, h.n_pool);
    if (rc == DSM_OK && info.store_cap > 0) rc = dsm_inactive_load(ctx, m.store, h.n_store, m.table, h.n_segments);
    if (rc != DSM_OK) return rc;
    if (h.extra_bytes > 0) std::memcpy(extra, m.extra, (size_t)h.extra_bytes);
    return DSM_OK;
}

extern "C" int dsm_map_peek(const char *path, void *extra, size_t extra_cap, size_t *extra_bytes, int32_t *kf_ofs_cnt, int seg_cap,
                            int *n_segments)
{
    if (!path || (extra_cap > 0 && !extra) || seg_cap < 0 || (seg_cap > 0 && !kf_ofs_cnt)) return DSM_E_INVALID;
    MapFile m;
    const int rc = m.read(path);
    if (rc != DSM_OK) return rc;
    if (extra_bytes) *extra_bytes = (size_t)m.hdr.extra_bytes;
    if (n_segments) *n_segments = m.hdr.n_segments;
    if (extra_cap > 0) std::memcpy(extra, m.extra, (size_t)std::min<uint64_t>(extra_cap, m.hdr.extra_bytes));
    if (seg_cap > 0) std::memcpy(kf_ofs_cnt, m.table, (size_t)std::min(seg_cap, m.hdr.n_segments) * 12);
    return DSM_OK;
}
