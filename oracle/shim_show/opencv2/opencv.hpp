// TEST INFRASTRUCTURE ONLY (oracle build).  oracle/shim/opencv2/opencv.hpp with an observable cv::imshow: placed before
// oracle/shim on the include path (oracle/show.mk), it includes that stand-in with its no-op imshow renamed away and
// defines an imshow that keeps a deep copy of the last image shown, so that a driver can read what the reference's
// debug_show() (fusion_functions.cpp:977-1006) displays.  No other oracle library is built with this directory.
#pragma once
#define imshow dsm_imshow_unused
#include "../../shim/opencv2/opencv.hpp"
#undef imshow

namespace cv
{
// the last image passed to imshow: rows x cols x elem bytes, packed rows
struct ShownImage
{
    std::string name;
    int rows = 0, cols = 0;
    size_t elem = 0;
    std::vector<uchar> bytes;
};
inline ShownImage &last_shown()
{
    static ShownImage s;
    return s;
}
inline void imshow(const char *name, const Mat &m)
{
    ShownImage &s = last_shown();
    s.name = name;
    s.rows = m.rows, s.cols = m.cols;
    s.elem = m.cols > 0 ? m.step / (size_t)m.cols : 0; // the images debug_show draws are owned, packed Mats
    s.bytes.resize((size_t)m.rows * m.cols * s.elem);
    for (int r = 0; r < m.rows; r++)
        memcpy(s.bytes.data() + (size_t)r * m.cols * s.elem, m.data + (size_t)r * m.step, (size_t)m.cols * s.elem);
}
} // namespace cv
