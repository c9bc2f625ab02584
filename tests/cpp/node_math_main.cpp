// Pins dsm::node_math (include/dsm_surfel_node.hpp) to the Eigen stand-in of the reference build (oracle/shim/Eigen):
// pose_ros2eigen, pose_eigen2ros, the 4x4 product, inverse and cast<float>, bit for bit on N random poses, both
// quaternion branches included.  Usage: node_math_main N; prints "N poses" and exits 0 when every value agrees.
#define DSM_SHIM_MAP_EXTRAS 1
#include <Eigen/Eigen> // oracle/shim
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include "dsm_surfel_node.hpp"

using dsm::node_math::M4;

static Eigen::Matrix4d ros2eigen(const dsm::Pose &p) // surfel_map.cpp:367-379 on the stand-in
{
    Eigen::Matrix4d T = Eigen::Matrix4d::Identity();
    Eigen::Quaterniond q;
    q.w() = p.qw, q.x() = p.qx, q.y() = p.qy, q.z() = p.qz;
    T.block<3, 3>(0, 0) = q.toRotationMatrix();
    T(0, 3) = p.x, T(1, 3) = p.y, T(2, 3) = p.z;
    return T;
}
static dsm::Pose eigen2ros(const Eigen::Matrix4d &T) // surfel_map.cpp:381-391 on the stand-in
{
    Eigen::Quaterniond q(T.block<3, 3>(0, 0));
    dsm::Pose p;
    p.qw = q.w(), p.qx = q.x(), p.qy = q.y(), p.qz = q.z();
    p.x = T(0, 3), p.y = T(1, 3), p.z = T(2, 3);
    return p;
}
static bool same(const double *a, const double *b, int n) { return std::memcmp(a, b, sizeof(double) * n) == 0; }

int main(int argc, char **argv)
{
    const int N = argc > 1 ? atoi(argv[1]) : 1000;
    std::mt19937_64 rng(7);
    std::normal_distribution<double> g(0.0, 1.0);
    int bad = 0;
    for (int n = 0; n < N; n++)
    {
        dsm::Pose a, b;
        double *pa[2] = {&a.x, &b.x};
        for (int k = 0; k < 2; k++)
        {
            double q[4], s = 0;
            for (int i = 0; i < 4; i++) s += (q[i] = g(rng)) * q[i];
            s = std::sqrt(s);
            if (n % 4 == 0) q[3] = 0.05 * q[3]; // rotations near 180 degrees: the largest-diagonal branch
            dsm::Pose &p = k ? b : a;
            p.x = 10 * g(rng), p.y = 10 * g(rng), p.z = 10 * g(rng);
            p.qx = q[0] / s, p.qy = q[1] / s, p.qz = q[2] / s, p.qw = q[3] / s;
        }
        (void)pa;
        const Eigen::Matrix4d ea = ros2eigen(a), eb = ros2eigen(b);
        const M4 ma = dsm::node_math::from_pose(a), mb = dsm::node_math::from_pose(b);
        const Eigen::Matrix4d eprod = ea * eb.inverse();
        const M4 mprod = dsm::node_math::mul(ma, dsm::node_math::inverse(mb));
        const dsm::Pose er = eigen2ros(eprod), mr = dsm::node_math::to_pose(mprod);
        const Eigen::Matrix4f ef = eprod.cast<float>();
        float mf[16];
        dsm::node_math::to_float(mprod, mf);
        const bool ok = same(ea.d, ma.d, 16) && same(eprod.d, mprod.d, 16) && same(&er.x, &mr.x, 7) &&
                        std::memcmp(ef.d, mf, sizeof(mf)) == 0;
        if (!ok && bad++ < 5) std::printf("pose %d differs\n", n);
    }
    if (bad) return 1;
    std::printf("%d poses\n", N);
    return 0;
}
