// dsm_context.hpp — the context owner of the header-only C++ classes (dsm::FusionFunctions, dsm::ResidentSurfelPool,
// dsm::SurfelMapNode): the dsm_ctx, the code of the last call and the one error report of the C++ layer, plus the
// read step of every map reader and the superpixel image.  Each class owns one detail::Context by value.  C++11.
#pragma once
#include <cstdio>
#include <cstring>
#include <type_traits>
#include <vector>
#include "dsm.h"

namespace dsm
{
namespace detail
{
class Context
{
  public:
    // owner: the class name that prefixes every message ("dsm::FusionFunctions", ...)
    explicit Context(const char *owner) : ctx(nullptr), err(DSM_OK), owner_(owner) {}
    ~Context() { close(); }
    Context(const Context &) = delete;
    Context &operator=(const Context &) = delete;

    static dsm_params params(int width, int height, float fx, float fy, float cx, float cy, float fuse_far, float fuse_near,
                             int max_batch, int max_local_surfels)
    {
        dsm_params p;
        std::memset(&p, 0, sizeof(p));
        p.width = width, p.height = height;
        p.fx = fx, p.fy = fy, p.cx = cx, p.cy = cy;
        p.fuse_far = fuse_far, p.fuse_near = fuse_near;
        p.max_batch = max_batch;
        p.max_local_surfels = max_local_surfels;
        return p;
    }

    // Replaces the context by a new one: dsm_create, then an empty resident pool when `resident`, an inactive store of
    // *max_inactive surfels when given and the constant set when given.  If any step fails, the failure is reported as
    // `what` and no context is left.
    int open(const char *what, const dsm_params &p, int device, bool resident, const int *max_inactive, const dsm_constants *constants)
    {
        close();
        int rc = dsm_create(&p, device, nullptr, &ctx);
        if (rc == DSM_OK && resident) rc = dsm_pool_upload(ctx, nullptr, 0);
        if (rc == DSM_OK && max_inactive) rc = dsm_inactive_reserve(ctx, *max_inactive);
        if (rc == DSM_OK && constants) rc = dsm_set_constants(ctx, constants);
        if (done(rc, what) != DSM_OK) close();
        return rc;
    }
    void close()
    {
        dsm_destroy(ctx);
        ctx = nullptr;
    }

    // true when there is a context; else the call `what` fails with DSM_E_STATE
    bool ready(const char *what)
    {
        if (ctx) return true;
        done(DSM_E_STATE, what);
        return false;
    }
    // the call `what`: op() when there is a context, else DSM_E_STATE, kept and reported by done()
    template <class Op>
    int run(const char *what, Op op)
    {
        return ready(what) ? done(op(), what) : err;
    }
    // keeps rc as the last error, reports it on stderr when it is not DSM_OK, and returns it
    int done(int rc, const char *what)
    {
        err = rc;
        if (rc != DSM_OK)
            std::fprintf(stderr, "%s::%s failed: %s (%s)\n", owner_, what, dsm_strerror(rc), ctx ? dsm_last_error(ctx) : "no context");
        return rc;
    }

    dsm_ctx *ctx;
    int err;

  private:
    const char *owner_;
};

// `in` appended to `out` field by field; both point types have float members x, y, z, intensity
template <class To, class From>
void append_points(std::vector<To> &out, const std::vector<From> &in)
{
    out.reserve(out.size() + in.size());
    for (size_t i = 0; i < in.size(); i++)
    {
        To p;
        p.x = in[i].x, p.y = in[i].y, p.z = in[i].z;
        p.intensity = in[i].intensity;
        out.push_back(p);
    }
}

// The read step of the C ABI's size-then-read: appends up to n records to `out` through read(records, cap, &n_out) and
// returns its code; on failure `out` is left as it was.  A caller type layout-identical to the ABI record Rec
// (dsm_surfel_t or the reference's SurfelElement, dsm_point_t or a 16-byte {x, y, z, intensity} POD) is read straight
// into `out`; a point type of other layout (pcl::PointXYZI) goes through dsm_point_t, converted field by field.
template <class Rec, class T, class Read>
int read_records(std::vector<T> &out, int n, Read read, std::true_type /* layout-identical */)
{
    const size_t base = out.size();
    out.resize(base + (size_t)n + 1); // one spare record: the buffer exists for n = 0
    int got = 0;
    const int rc = read(reinterpret_cast<Rec *>(&out[base]), n, &got);
    out.resize(rc == DSM_OK ? base + (size_t)got : base);
    return rc;
}
template <class Rec, class T, class Read>
int read_records(std::vector<T> &out, int n, Read read, std::false_type)
{
    static_assert(std::is_same<Rec, dsm_point_t>::value, "SurfelElement must be the 44-byte reference POD");
    std::vector<Rec> recs;
    const int rc = read_records<Rec>(recs, n, read, std::true_type());
    append_points(out, recs);
    return rc;
}
template <class Rec, class T, class Read>
int read_records(std::vector<T> &out, int n, Read read)
{
    return read_records<Rec>(out, n, read, std::integral_constant<bool, sizeof(T) == sizeof(Rec)>());
}

// FusionFunctions::debug_show (fusion_functions.cpp:977-1006) of the last fused frame into a caller's image: any type
// with .data and .step (a cv::Mat of CV_8UC3)
template <class Mat>
int superpixel_image(Context &c, Mat &image)
{
    return dsm_frame_superpixel_image(c.ctx, 0, reinterpret_cast<uint8_t *>(image.data), (size_t)image.step);
}
} // namespace detail
} // namespace dsm
