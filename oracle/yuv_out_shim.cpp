// TEST INFRASTRUCTURE - the reference's RGBA8 -> YUV conversion (core/src/image.cpp:1051-1100: rgba8ToNv12, rgba8ToNv21, rgba8ToI420)
// as plain C symbols: the reference's own libyuv entry points ABGRToNV12 / ABGRToNV21 / ABGRToI420, compiled with the portable C rows
// of its vendored libyuv (see yuv_out.mk). Every function reads RGBA8 (libyuv's "ABGR") rows of `src_pitch` bytes and returns libyuv's
// status.
#include "libyuv/convert.h"
#include "libyuv/convert_from_argb.h"

using namespace libyuv;

extern "C" {
int yuv_rgba_to_nv12(const uint8_t* src, int src_pitch, uint8_t* y, int py, uint8_t* uv, int puv, int w, int h) {
    return ABGRToNV12(src, src_pitch, y, py, uv, puv, w, h);
}
int yuv_rgba_to_nv21(const uint8_t* src, int src_pitch, uint8_t* y, int py, uint8_t* vu, int pvu, int w, int h) {
    return ABGRToNV21(src, src_pitch, y, py, vu, pvu, w, h);
}
int yuv_rgba_to_i420(const uint8_t* src, int src_pitch, uint8_t* y, int py, uint8_t* u, int pu, uint8_t* v, int pv, int w, int h) {
    return ABGRToI420(src, src_pitch, y, py, u, pu, v, pv, w, h);
}
}
