// TEST INFRASTRUCTURE ONLY.  The serial reference oracle of ref_driver.cpp (the reference's own fusion_functions.cpp
// compiled in place, thread bodies inline) with one more hook, for FusionFunctions::debug_show (fusion_functions.cpp:
// 977-1006), the superpixel normal image the reference draws and hands to cv::imshow.  Built into
// oracle/_ref/libdsm_ref_show.so by oracle/Makefile against oracle/shim_show, whose imshow keeps the last image shown;
// every entry point of libdsm_ref_serial.so is exported too.
#include "ref_driver.cpp"

extern "C"
{
    // debug_show() on the context's superpixel_index / superpixel_seeds, after overwriting them with labels[H*W] /
    // seeds[S] (60-byte Superpixel_seed records) where those are non-null.  Writes the [H][W][3] bytes it showed to
    // out_bgr; returns 0, or -1 when nothing of that shape was shown.
    int dsmref_debug_show(void *p, const int32_t *labels, const void *seeds, uint8_t *out_bgr)
    {
        RefCtx *c = (RefCtx *)p;
        if (labels) memcpy(c->ff.superpixel_index.data(), labels, c->ff.superpixel_index.size() * sizeof(int));
        if (seeds) memcpy((void *)c->ff.superpixel_seeds.data(), seeds, c->ff.superpixel_seeds.size() * sizeof(Superpixel_seed));
        cv::last_shown() = cv::ShownImage();
        c->ff.debug_show();
        const cv::ShownImage &s = cv::last_shown();
        if (s.rows != c->h || s.cols != c->w || s.elem != 3) return -1;
        memcpy(out_bgr, s.bytes.data(), s.bytes.size());
        return 0;
    }
}
