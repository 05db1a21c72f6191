// png++/png.hpp -- stand-in for png++ used only when tests/golden/make_ref_obj.py compiles the reference's train_obj.cpp.
// It comes before oracle/shim on the include path.  An image "loaded" from a path is the pixel buffer the harness
// registered under that path (BGR or 16-bit depth, tests/golden/ref_obj/ref_train_obj.cpp); an unregistered path is a
// black 640x480 frame, as in oracle/shim/png++/png.hpp.
#pragma once
#include <cstdint>
#include <string>

extern "C" int ref_obj_png_lookup(const char* path, int* width, int* height, const uint8_t** bgr, const uint16_t** depth);

namespace png {
template <typename T> struct basic_rgb_pixel {
    T red, green, blue;
    basic_rgb_pixel() : red(0), green(0), blue(0) {}
};

template <typename Pixel> struct pixel_of;
template <> struct pixel_of<unsigned short> {
    static unsigned short get(const uint8_t*, const uint16_t* d, int i) { return d ? d[i] : 0; }
};
template <typename T> struct pixel_of<basic_rgb_pixel<T>> {
    static basic_rgb_pixel<T> get(const uint8_t* b, const uint16_t*, int i) {
        basic_rgb_pixel<T> p;
        if (b) { p.blue = b[3 * i]; p.green = b[3 * i + 1]; p.red = b[3 * i + 2]; }
        return p;
    }
};

template <typename Pixel> class image {
public:
    explicit image(const std::string& path) : w_(640), h_(480), bgr_(nullptr), depth_(nullptr) {
        ref_obj_png_lookup(path.c_str(), &w_, &h_, &bgr_, &depth_);
    }
    int get_width() const { return w_; }
    int get_height() const { return h_; }
    Pixel get_pixel(int x, int y) const { return pixel_of<Pixel>::get(bgr_, depth_, y * w_ + x); }

private:
    int w_, h_;
    const uint8_t* bgr_;
    const uint16_t* depth_;
};
}  // namespace png
