// Shared by the C++ test drivers of this directory: the reference's caller types, the binary I/O of a driver's in.bin
// and out.bin, the frame record of the fuse_map drivers, the harness of the node drivers (argument prefix, message loop,
// cloud records and digest), and the pieces of the known-field node drivers (field arguments, the field handout of each
// depth message, the reload step and the end of a drive).  Every record is read and written in the layout the driver's
// header comment gives.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <initializer_list>
#include <string>
#include <vector>
#include <opencv2/opencv.hpp> // oracle/shim
#include "dsm_surfel_node.hpp"

struct SurfelElement // reference elements.h:22-31
{
    float px, py, pz, nx, ny, nz, size, color, weight;
    int update_times, last_update;
};
struct PointXYZI // the four named fields of pcl::PointXYZI
{
    float x, y, z, intensity;
};
struct Pose4f // Eigen::Matrix4f: a column-major .data()
{
    float m[16];
    float *data() { return m; }
};

static FILE *in_f, *out_f; // the driver's in.bin and out.bin

// false (exit code 5) when either file cannot be opened
inline bool open_io(const char *in, const char *out)
{
    in_f = fopen(in, "rb");
    out_f = fopen(out, "wb");
    return in_f && out_f;
}
inline int close_io()
{
    fclose(in_f);
    fclose(out_f);
    return 0;
}

// the exit code of a set-up error (last_error() after construction): 0 for none, 3 when there is no usable GPU (the
// library has no CPU fallback), 4 for any other
inline int setup_code(int last_error)
{
    return last_error == DSM_OK ? 0 : last_error == DSM_E_NODEVICE ? 3 : 4;
}

template <class T>
static bool get(T &v)
{
    return fread(&v, sizeof(T), 1, in_f) == 1;
}
template <class T>
static bool get_n(std::vector<T> &v, int n)
{
    if (n < 0) return false;
    v.resize((size_t)n);
    return n == 0 || fread(v.data(), sizeof(T), (size_t)n, in_f) == (size_t)n;
}
template <class T>
static void put(const T &v)
{
    fwrite(&v, sizeof(T), 1, out_f);
}
// int32 n, then n records
template <class T>
static void put_n(const T *p, int n)
{
    put(n);
    if (n > 0) fwrite(p, sizeof(T), (size_t)n, out_f);
}
template <class T>
static void put_list(const std::vector<T> &v)
{
    put_n(v.data(), (int)v.size());
}

// one frame of the fuse_map drivers: int32 ref_idx, float pose[16], then (after what the driver reads in between)
// uint8 gray[H*W], float depth[H*W]; image() and depth_map() are cv::Mat views of the two planes
struct FrameRecord
{
    int W, H, ref;
    Pose4f pose;
    std::vector<unsigned char> gray;
    std::vector<float> depth;
    FrameRecord(int w, int h) : W(w), H(h), ref(0) {}
    bool get_head() { return get(ref) && get(pose); }
    bool get_images() { return get_n(gray, W * H) && get_n(depth, W * H); }
    cv::Mat image() { return cv::Mat(H, W, CV_8UC1, gray.data(), (size_t)W); }
    cv::Mat depth_map() { return cv::Mat(H, W, CV_32FC1, depth.data(), (size_t)W * 4); }
};

// The orb / image / depth messages of the node drivers' script (node_main.cpp), each handed to the node as it is read:
//   0 orb    double stamp, int32 is_keyframe, int32 reference_index, double pose7[7], int32 n_path, double path7[n_path][7],
//            int32 n_loops, int32 pairs[2 n_loops]
//   1 image  double stamp, uint8 gray[H*W]
//   2 depth  double stamp, float depth[H*W]
struct NodeMessages
{
    std::vector<uint8_t> gray;
    std::vector<float> depth;
    std::vector<double> path;
    std::vector<int> pairs;
    // false for a malformed message or another type; else rc is the node's code
    template <class Node>
    bool feed(Node &node, int type, int W, int H, int &rc)
    {
        double stamp = 0;
        if (type == 0)
        {
            int kf = 0, ref = 0, n_path = 0, n_loops = 0;
            double pose[7];
            if (!get(stamp) || !get(kf) || !get(ref) || fread(pose, 8, 7, in_f) != 7 || !get(n_path) || !get_n(path, 7 * n_path) ||
                !get(n_loops) || !get_n(pairs, 2 * n_loops))
                return false;
            rc = node.orb_results_input(stamp, pairs.data(), n_loops, path.data(), n_path, pose, kf != 0, ref);
        }
        else if (type == 1)
        {
            if (!get(stamp) || !get_n(gray, W * H)) return false;
            rc = node.image_input(stamp, gray.data(), (size_t)W);
        }
        else if (type == 2)
        {
            if (!get(stamp) || !get_n(depth, W * H)) return false;
            rc = node.depth_input(stamp, depth.data(), (size_t)W * 4);
        }
        else
            return false;
        return true;
    }
    // one message to node a, then the same message to node b
    template <class Node>
    bool feed_both(Node &a, Node &b, int type, int W, int H, int &ra, int &rb)
    {
        const long at = ftell(in_f);
        if (!feed(a, type, W, H, ra)) return false;
        fseek(in_f, at, SEEK_SET);
        return feed(b, type, W, H, rb);
    }
};

// ---- the node drivers ----

// The argument prefix of the node drivers: argv[1..9] = W H fx fy cx cy far near drift_free_poses, then, in the drivers
// that take them, argv[10..12] = device max_local max_inactive (else device 0, 2^20 pool and 2^21 stored surfels).
struct NodeArgs
{
    int W, H, dfp, device, max_local, max_inactive;
    double fx, fy, cx, cy, fr, nr;
    NodeArgs(char **argv, bool sized)
        : W(atoi(argv[1])), H(atoi(argv[2])), dfp(atoi(argv[9])), device(sized ? atoi(argv[10]) : 0),
          max_local(sized ? atoi(argv[11]) : 1 << 20), max_inactive(sized ? atoi(argv[12]) : 1 << 21), fx(atof(argv[3])),
          fy(atof(argv[4])), cx(atof(argv[5])), cy(atof(argv[6])), fr(atof(argv[7])), nr(atof(argv[8]))
    {
    }
};

// a node of the prefix's parameters; check setup_code(last_error())
struct DriverNode : dsm::SurfelMapNode
{
    explicit DriverNode(const NodeArgs &a, const dsm_constants *constants = nullptr)
        : dsm::SurfelMapNode(a.W, a.H, a.fx, a.fy, a.cx, a.cy, a.fr, a.nr, a.dfp, a.device, a.max_local, a.max_inactive, constants)
    {
    }
};

// Feeds the script's orb / image / depth messages to the node until its end and calls on_depth() after every depth
// message.  Returns 0 at the end, 5 for a malformed message, 6 when the node refuses one, else the first nonzero code
// on_depth() returns.
template <class F>
static int feed_script(dsm::SurfelMapNode &node, int W, int H, F on_depth)
{
    NodeMessages msg;
    int type = 0, r = DSM_OK;
    while (get(type))
    {
        if (!msg.feed(node, type, W, H, r)) return 5;
        if (r != DSM_OK) return 6;
        if (type != 2) continue;
        const int e = on_depth();
        if (e) return e;
    }
    return 0;
}

// int32 rc, then the clouds of active_points() and inactive_points() (each int32 n + n points).  inactive_points() is
// read only after active_points() succeeded; after a failed read the inactive cloud written is the previous one.
inline void put_clouds(dsm::SurfelMapNode &node)
{
    static std::vector<dsm_point_t> act, inact;
    int rc = node.active_points(act);
    if (rc == DSM_OK) rc = node.inactive_points(inact);
    put(rc);
    put_list(act);
    put_list(inact);
}

// the end of a drive: local_surfels (int32 n + records) and inactive_points; false (exit code 6) when a read fails
inline bool put_final(dsm::SurfelMapNode &node)
{
    std::vector<dsm_surfel_t> local;
    std::vector<dsm_point_t> inact;
    if (node.local_surfels(local) != DSM_OK || node.inactive_points(inact) != DSM_OK) return false;
    put_list(local);
    put_list(inact);
    return true;
}

// save_mesh to <prefix>.ply and save_cloud to <prefix>.pcd; false (exit code 6) when either fails
inline bool save_files(dsm::SurfelMapNode &node, const std::string &prefix)
{
    return node.save_mesh(prefix + ".ply") == DSM_OK && node.save_cloud(prefix + ".pcd") == DSM_OK;
}

// ---- the known-field node drivers ----

// The field block of their arguments, argv[13..18] = voxel nx ny nz max_views max_range, after the sized prefix.
struct FieldArgs
{
    float voxel, max_range;
    int nx, ny, nz, max_views;
    explicit FieldArgs(char **argv)
        : voxel((float)atof(argv[13])), max_range((float)atof(argv[18])), nx(atoi(argv[14])), ny(atoi(argv[15])), nz(atoi(argv[16])),
          max_views(atoi(argv[17]))
    {
    }
    int cells() const { return nx * ny * nz; }
    // enable_distance_field, then enable_known_space unless max_views is 0; 4 when either fails
    int enable(dsm::SurfelMapNode &node) const
    {
        if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
        if (max_views > 0 && node.enable_known_space(max_views, max_range) != DSM_OK) return 4;
        return 0;
    }
    // the centre of the grid's middle voxel, ((origin + n / 2) + 0.5) * voxel per axis
    void middle(const int32_t origin[3], double c[3]) const
    {
        const int n[3] = {nx, ny, nz};
        for (int a = 0; a < 3; a++) c[a] = ((double)(origin[a] + n[a] / 2) + 0.5) * (double)voxel;
    }
};

// The field of the frame just fused: distance_field(), then, with `known`, known_space() when distance_field() handed
// out a field (DSM_OK, and with `capacity` DSM_E_CAPACITY too).  rs is rc when known_space() was not called.
struct FieldHandout
{
    const float *dist;
    const uint8_t *state;
    int32_t origin[3];
    int n_occ, n_free, rc, rs;
    FieldHandout(dsm::SurfelMapNode &node, bool known, bool capacity = false) : dist(nullptr), state(nullptr), n_occ(0), n_free(0)
    {
        origin[0] = origin[1] = origin[2] = 0;
        rc = node.distance_field(dist, origin, n_occ);
        rs = known && (rc == DSM_OK || (capacity && rc == DSM_E_CAPACITY)) ? node.known_space(state, n_free) : rc;
    }
    bool ok() const { return rc == DSM_OK && rs == DSM_OK; }
    void put_origin() const { put(origin[0]), put(origin[1]), put(origin[2]); }
    // the grids (int32 n + n values), empty unless ok()
    void put_state(const FieldArgs &f) const { put_n(state, ok() ? f.cells() : 0); }
    void put_dist(const FieldArgs &f) const { put_n(dist, ok() ? f.cells() : 0); }
};

// the first code of a chain of calls that is not DSM_OK, else DSM_OK
inline int first_error(std::initializer_list<int> rcs)
{
    for (int rc : rcs)
        if (rc != DSM_OK) return rc;
    return DSM_OK;
}

// save_state and load_state through <prefix>.state; false (exit code 6) when either fails
inline bool reload(dsm::SurfelMapNode &node, const std::string &prefix)
{
    return node.save_state(prefix + ".state") == DSM_OK && node.load_state(prefix + ".state") == DSM_OK;
}

// the end of a drive: local_surfels (int32 n + records), save_mesh and save_cloud to <prefix>.ply / .pcd, then the
// files closed; 6 when a read or a save fails, else 0
inline int end_drive(dsm::SurfelMapNode &node, const std::string &prefix)
{
    std::vector<dsm_surfel_t> local;
    if (node.local_surfels(local) != DSM_OK) return 6;
    put_list(local);
    if (!save_files(node, prefix)) return 6;
    return close_io();
}

template <class T>
static void add(std::vector<uint8_t> &d, const T *p, size_t n)
{
    const uint8_t *b = reinterpret_cast<const uint8_t *>(p);
    d.insert(d.end(), b, b + n * sizeof(T));
}
template <class T>
static void add_list(std::vector<uint8_t> &d, const std::vector<T> &v)
{
    const int n = (int)v.size();
    add(d, &n, 1);
    add(d, v.data(), v.size());
}

// everything the node reads back, as bytes: local_surfels, attached_surfels of every pose, poses() (cam_pose,
// loop_pose, cam_stamp, links), local_surfels_indexs(), pending_frame(), last_warp() and pose_graph()
inline std::vector<uint8_t> digest(dsm::SurfelMapNode &node)
{
    std::vector<uint8_t> d;
    std::vector<dsm_surfel_t> s;
    int rc = node.local_surfels(s);
    add(d, &rc, 1);
    add_list(d, s);
    const std::vector<dsm::NodePose> &p = node.poses();
    for (size_t i = 0; i < p.size(); i++)
    {
        rc = node.attached_surfels((int)i, s);
        add(d, &rc, 1);
        add_list(d, s);
        add(d, &p[i].cam_pose, 1);
        add(d, &p[i].loop_pose, 1);
        add(d, &p[i].cam_stamp, 1);
        add_list(d, p[i].linked_pose_index);
    }
    add_list(d, std::vector<int>(node.local_surfels_indexs().begin(), node.local_surfels_indexs().end()));
    float pose16[16] = {0};
    std::vector<int> rem, add_;
    const int pref = node.pending_frame(pose16, rem, add_);
    add(d, &pref, 1);
    add(d, pose16, 16);
    add_list(d, rem);
    add_list(d, add_);
    add_list(d, node.last_warp());
    const dsm::NodePoseGraph g = node.pose_graph();
    add_list(d, g.path);
    add_list(d, g.loop_edges);
    add_list(d, g.driftfree);
    add_list(d, g.drift);
    add(d, &g.camera, 1);
    return d;
}
