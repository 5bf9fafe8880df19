// TEST INFRASTRUCTURE - the reference's colour conversion (core/src/image.cpp:1076-1136: nv12ToRgba8, nv21ToRgba8, i420ToRgba8) as
// plain C symbols, compiled with the portable C rows of the reference's vendored libyuv (see yuv.mk). Every function writes RGBA8
// (libyuv's "ABGR") rows of `dst_pitch` bytes and returns libyuv's status.
//
// BT.601 calls the reference's own entry points. For BT.709, I420 calls H420ToABGR; this libyuv exports no BT.709 form of NV12ToABGR /
// NV21ToABGR (NV21ToARGBMatrix / NV12ToARGBMatrix are file-static), so nv_rows() drives libyuv's C rows with kYvuH709Constants the way
// those functions do: one row per luma row, the chroma row advancing after every odd row. `bt709 == 2` runs nv_rows() with
// kYvuI601Constants, so that the tests can hold it to the public BT.601 entry points.
#include "libyuv/convert_argb.h"
#include "libyuv/row.h"

using namespace libyuv;

typedef void (*NvRow)(const uint8_t*, const uint8_t*, uint8_t*, const struct YuvConstants*, int);
static int nv_rows(NvRow row, const uint8_t* y, int py, const uint8_t* c, int pc, uint8_t* dst, int dst_pitch, const struct YuvConstants* k, int w, int h) {
    if (!y || !c || !dst || w <= 0 || h <= 0) return -1;
    for (int r = 0; r < h; ++r) {
        row(y, c, dst, k, w);
        y += py, dst += dst_pitch;
        if (r & 1) c += pc;
    }
    return 0;
}

extern "C" {
// NV12ToABGR = NV21ToARGBMatrix(kYvuI601Constants): the UV plane read through the VU row with the swapped table
int yuv_nv12_to_rgba(const uint8_t* y, int py, const uint8_t* uv, int puv, uint8_t* dst, int dst_pitch, int w, int h, int bt709) {
    if (bt709) return nv_rows(NV21ToARGBRow_C, y, py, uv, puv, dst, dst_pitch, bt709 == 2 ? &kYvuI601Constants : &kYvuH709Constants, w, h);
    return NV12ToABGR(y, py, uv, puv, dst, dst_pitch, w, h);
}
int yuv_nv21_to_rgba(const uint8_t* y, int py, const uint8_t* vu, int pvu, uint8_t* dst, int dst_pitch, int w, int h, int bt709) {
    if (bt709) return nv_rows(NV12ToARGBRow_C, y, py, vu, pvu, dst, dst_pitch, bt709 == 2 ? &kYvuI601Constants : &kYvuH709Constants, w, h);
    return NV21ToABGR(y, py, vu, pvu, dst, dst_pitch, w, h);
}
int yuv_i420_to_rgba(const uint8_t* y, int py, const uint8_t* u, int pu, const uint8_t* v, int pv, uint8_t* dst, int dst_pitch, int w, int h, int bt709) {
    return bt709 ? H420ToABGR(y, py, u, pu, v, pv, dst, dst_pitch, w, h) : I420ToABGR(y, py, u, pu, v, pv, dst, dst_pitch, w, h);
}
}
